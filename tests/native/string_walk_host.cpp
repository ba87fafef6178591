// string_walk_host.cpp - compiles the string_val walk of the concatenated string decode (min-tfs-client_b200/csrc/string_walk.h)
// for the HOST, composed the way str_index_kernel composes it (the output's last `value` occurrence, at most n_strings entries),
// so that tests/test_concat_strings_cpu.py can hold it against the protobuf runtime without a GPU.  Test infrastructure only.
#include "../../min-tfs-client_b200/csrc/string_walk.h"

using namespace b200tfs;

namespace {
struct Collect {
  uint64_t* off; uint32_t* len; uint64_t cap;
  void operator()(uint64_t j, uint32_t o, uint32_t n) {
    if (j < cap) { off[j] = o; len[j] = n; }
  }
};
}  // namespace

extern "C" {

// The string_val elements of the TensorProto at [msg_off, msg_off + msg_len) of a record: their record-relative offsets and
// lengths (at most cap), their count in *count.  Returns B200TFS_OK or the walk's error.
int sw_strings(const uint8_t* rec, uint64_t rec_len, uint64_t msg_off, uint64_t msg_len, uint64_t* off, uint32_t* len, uint64_t cap,
               uint64_t* count) {
  *count = 0;
  if (rec_len > 0x7FFFFFFFull || msg_off + msg_len > rec_len) return B200TFS_E_ARG;
  Cursor c;
  cur_open_host(c, rec, (uint32_t)rec_len);
  c.p = (uint32_t)msg_off;
  c.end = (uint32_t)(msg_off + msg_len);
  Collect s{off, len, cap};
  *count = walk_strings(c, s);
  return c.err ? c.err : B200TFS_OK;
}

uint64_t sw_count_bound(uint64_t rec_len) { return str_count_bound(rec_len); }

}  // extern "C"
