// example_walk_host.cpp - compiles the Classify / Regress response walk (min-tfs-client_b200/csrc/example_walk.h) for the HOST,
// composed the way the kernels compose it (index: entries; emit: every entry's value or classes), so that
// tests/test_example_response_walk_cpu.py can hold it against the protobuf runtime without a GPU.  Test infrastructure only.
#include <vector>

#include "../../min-tfs-client_b200/csrc/example_walk.h"

using namespace b200tfs;

namespace {
struct Entries {
  std::vector<b200tfs_label_ref> e;
  void operator()(uint32_t off, uint32_t len) { e.push_back(b200tfs_label_ref{off, len}); }
};
struct Count {
  void operator()(uint32_t, uint32_t, uint32_t, uint32_t) {}
};
struct Store {
  uint32_t* values; b200tfs_label_ref* labels;
  uint64_t base, C, cap;
  void operator()(uint32_t k, uint32_t off, uint32_t len, uint32_t score) {
    if (k >= C || base + k >= cap) return;
    values[base + k] = score;
    labels[base + k] = b200tfs_label_ref{off, len};
  }
};
}  // namespace

extern "C" {

// One response of `kind` (B200TFS_RESP_*).  Classify: C < 0 lets the response's first example set the class count.  values /
// labels (Classify) receive row-major entries below `cap`.  Returns B200TFS_OK, B200TFS_E_PARSE or B200TFS_E_SHAPE (an example
// with another class count); *rows and *n_classes as the kernels find them.
int xw_decode(int kind, const uint8_t* wire, uint64_t len, int64_t C, float* values, b200tfs_label_ref* labels, uint64_t cap,
              uint64_t* rows, int64_t* n_classes, b200tfs_model_spec* spec) {
  *rows = 0;
  *n_classes = 0;
  if (len > 0x7FFFFFFFull) return B200TFS_E_PARSE;
  Cursor c;
  cur_open_host(c, wire, (uint32_t)len);
  Entries ent;
  if (xr_walk_response(c, *spec, ent)) return B200TFS_E_PARSE;
  *rows = ent.e.size();
  uint32_t* v = reinterpret_cast<uint32_t*>(values);
  bool shape = false;
  if (kind == B200TFS_RESP_CLASSIFY && C < 0) {
    C = 0;
    if (!ent.e.empty()) {
      c.p = ent.e[0].off; c.end = ent.e[0].off + ent.e[0].len;
      Count cnt;
      C = xr_classes(c, cnt);
      c.err = 0;
    }
  }
  for (size_t i = 0; i < ent.e.size(); ++i) {
    c.p = ent.e[i].off; c.end = ent.e[i].off + ent.e[i].len; c.err = 0;
    if (kind == B200TFS_RESP_REGRESS) {
      const uint32_t x = xr_regression(c);
      if (c.err) return B200TFS_E_PARSE;
      if (i < cap) v[i] = x;
    } else {
      Store s{v, labels, i * (uint64_t)C, (uint64_t)C, cap};
      const uint32_t k = xr_classes(c, s);
      if (c.err) return B200TFS_E_PARSE;
      shape = shape || k != (uint64_t)C;
    }
  }
  *n_classes = kind == B200TFS_RESP_CLASSIFY ? C : 0;
  return shape ? B200TFS_E_SHAPE : B200TFS_OK;
}

uint64_t xw_row_bound(uint64_t len) { return xr_row_bound(len); }
}
