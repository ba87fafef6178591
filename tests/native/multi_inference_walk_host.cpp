// multi_inference_walk_host.cpp - compiles the MultiInference response walk (min-tfs-client_b200/csrc/multi_walk.h) for the HOST,
// composed the way the kernels compose it (index: each result's entries to its task; per task, emit: every entry's value or
// classes), so that tests/test_multi_inference_cpu.py can hold it against the protobuf runtime without a GPU.  Test infrastructure
// only.
#include <vector>

#include "../../min-tfs-client_b200/csrc/multi_walk.h"

using namespace b200tfs;

namespace {
struct Entries {
  std::vector<b200tfs_label_ref>* e;
  void operator()(uint32_t off, uint32_t len) { e->push_back(b200tfs_label_ref{off, len}); }
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

// One response of a request whose n_tasks tasks have kinds[t] (B200TFS_RESP_*).  Task t writes its values (Classify: row-major
// scores, and labels) from values + t * cap / labels + t * cap, below cap; status[t], rows[t], n_classes[t] and specs[t] as the
// kernels leave them for this response.
void mw_decode(int n_tasks, const int* kinds, const uint8_t* wire, uint64_t len, float* values, b200tfs_label_ref* labels,
               uint64_t cap, int* status, uint64_t* rows, int64_t* n_classes, b200tfs_model_spec* specs) {
  std::vector<std::vector<b200tfs_label_ref>> ent(n_tasks);
  std::vector<int> match(n_tasks, 0);
  for (int t = 0; t < n_tasks; ++t) { rows[t] = 0; n_classes[t] = 0; spec_reset(specs[t]); }
  if (len > 0x7FFFFFFFull) { for (int t = 0; t < n_tasks; ++t) status[t] = B200TFS_E_PARSE; return; }
  Cursor c;
  cur_open_host(c, wire, (uint32_t)len);
  uint32_t k = 0, lo, hi;
  while (!c.err && mi_next_result(c, &lo, &hi)) {
    b200tfs_model_spec spec;
    spec_reset(spec);
    uint32_t kase, from;
    mi_result_case(c, lo, hi, spec, &kase, &from);
    if (c.err) break;
    if (k >= (uint32_t)n_tasks || kase != mi_case_of((uint32_t)kinds[k])) {
      mi_check_run(c, kase, from, hi);
    } else {
      match[k] = 1;
      Cursor d = c;
      d.p = from; d.end = hi;
      uint32_t blo, bhi;
      Entries on{&ent[k]};
      while (!c.err && mi_next_member(d, kase, &blo, &bhi)) xr_entries(c, blo, bhi, on);
    }
    if (k < (uint32_t)n_tasks) specs[k] = spec;
    ++k;
  }
  const int err = c.err;
  for (int t = 0; t < n_tasks; ++t) {
    if (err) { status[t] = B200TFS_E_PARSE; spec_reset(specs[t]); continue; }
    status[t] = k != (uint32_t)n_tasks || !match[t] ? B200TFS_E_SHAPE : B200TFS_OK;
    if (!match[t]) continue;
    const std::vector<b200tfs_label_ref>& e = ent[t];
    rows[t] = e.size();
    uint32_t* v = reinterpret_cast<uint32_t*>(values + (uint64_t)t * cap);
    b200tfs_label_ref* lb = labels + (uint64_t)t * cap;
    uint64_t C = 0;
    if (kinds[t] == B200TFS_RESP_CLASSIFY && !e.empty()) {
      c.p = e[0].off; c.end = e[0].off + e[0].len; c.err = 0;
      Count cnt;
      C = xr_classes(c, cnt);
    }
    n_classes[t] = (int64_t)C;
    int st = B200TFS_OK;
    for (size_t i = 0; i < e.size(); ++i) {
      c.p = e[i].off; c.end = e[i].off + e[i].len; c.err = 0;
      if (kinds[t] == B200TFS_RESP_REGRESS) {
        const uint32_t x = xr_regression(c);
        if (c.err) { st = B200TFS_E_PARSE; break; }
        if (i < cap) v[i] = x;
      } else {
        Store s{v, lb, i * C, C, cap};
        const uint32_t got = xr_classes(c, s);
        if (c.err) { st = B200TFS_E_PARSE; break; }
        if (got != C && st == B200TFS_OK) st = B200TFS_E_SHAPE;
      }
    }
    if (st != B200TFS_OK && (status[t] == B200TFS_OK || st < status[t])) status[t] = st;
  }
}

uint64_t mw_row_bound(uint64_t rec_len) { return xr_row_bound(rec_len); }

}  // extern "C"
