// string_walk.h - the string_val walk of one TensorProto (tensor.proto: repeated bytes string_val = 8) that the concatenated
// string decode runs three times over: the host layout (b200tfs_concat_strings_layout) counts strings and bytes with it, the index
// kernel (string_kernels.cuh) records where each string lies, and tests/native replays responses and mutants of them through it.
// Built from walker.h's cursor, tag, length and skip helpers, so it reads the wire exactly as the parse kernel's walk_tensor does.
#pragma once
#include "walker.h"

namespace b200tfs {

// Every string_val element takes at least its tag and its length byte, and its bytes lie in the wire: one output of a record of
// L bytes holds at most L / 2 strings of at most L bytes in all.
B2_HD uint64_t str_count_bound(uint64_t rec_len) { return rec_len / 2; }

// The string_val elements of the TensorProto body [c.p, c.end), in wire order: sink(j, off, len) for element j, `off` the
// record-relative offset of its first byte.  Every other field is skipped.  Returns the elements found; an error stays in c.err.
template <class Sink>
B2_HD uint64_t walk_strings(Cursor& c, Sink& sink) {
  uint64_t j = 0;
#pragma unroll 1
  while (c.p < c.end && !c.err) {
    const uint32_t tag = rd_tag(c);
    if (c.err) break;
    if (tag != tag_of(F_STRING, WT_LEN)) { skip_field(c, tag); continue; }
    const uint32_t n = rd_len(c);
    if (c.err) break;
    sink(j++, c.p, n);
    c.p += n;
  }
  return j;
}

}  // namespace b200tfs
