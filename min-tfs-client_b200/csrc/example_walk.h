// example_walk.h - the ClassificationResponse / RegressionResponse walk (classification.proto, regression.proto) that the
// example-response kernels run (example_resp_kernels.cuh), built from walker.h's cursor, skip, varint and UTF-8 helpers.  The
// same source compiles for the host, where tests/native replays responses and mutants of them through it.
//
//   {Classification,Regression}Response { result = 1; model_spec = 2; }
//   ClassificationResult { repeated Classifications classifications = 1; }   RegressionResult { repeated Regression regressions = 1; }
//   Classifications { repeated Class classes = 1; }   Class { string label = 1; float score = 2; }   Regression { float value = 1; }
//
// What the runtime does, and so what the walk does: fields in any order; the last of a repeated scalar wins; unknown fields
// (groups included) are skipped at every level; a known field with another wire type is an unknown field; repeated `result`
// and `model_spec` fields merge (the result's entries concatenate); labels must be UTF-8 (proto3 string).
#pragma once
#include "walker.h"

namespace b200tfs {

// Every Regression, Classifications and Class entry takes at least its tag and its length byte: a record of L bytes holds at
// most L / 2 rows, and one example at most L / 2 classes.
B2_HD uint64_t xr_row_bound(uint64_t rec_len) { return rec_len / 2; }

// The top level from c.p on, up to the next `result` field: model_spec occurrences merge into *spec, other fields are skipped.
// Returns true with the result's body in [*lo, *hi) (the cursor behind it), false at the end of the record or on an error.
B2_HD bool xr_next_result(Cursor& c, b200tfs_model_spec& spec, uint32_t* lo, uint32_t* hi) {
#pragma unroll 1
  while (c.p < c.end && !c.err) {
    const uint32_t tag = rd_tag(c);
    if (c.err) break;
    if (tag == tag_of(1, WT_LEN)) {            // result
      const uint32_t m = rd_len(c);
      if (c.err) break;
      *lo = c.p; *hi = c.p + m;
      c.p += m;
      return true;
    }
    if (tag == tag_of(2, WT_LEN)) {            // model_spec
      const uint32_t m = rd_len(c);
      if (c.err) break;
      const uint32_t outer = c.end;
      c.end = c.p + m;
      walk_model_spec(c, spec);
      c.end = outer;
    } else skip_field(c, tag);
  }
  return false;
}

// Every field of the message body [lo, hi) in turn: on_entry(off, len) for each field-1 sub-message (a Regression, a
// Classifications or a Class), every other field skipped.  Leaves an error in c.err; the cursor's range is restored.
template <class OnEntry>
B2_HD void xr_entries(Cursor& c, uint32_t lo, uint32_t hi, OnEntry& on_entry) {
  const uint32_t p0 = c.p, outer = c.end;
  c.p = lo; c.end = hi;
#pragma unroll 1
  while (c.p < c.end && !c.err) {
    const uint32_t t = rd_tag(c);
    if (c.err) break;
    if (t == tag_of(1, WT_LEN)) {
      const uint32_t n = rd_len(c);
      if (c.err) break;
      on_entry(c.p, n);
      c.p += n;
    } else skip_field(c, t);
  }
  c.p = p0; c.end = outer;
}

// One response's top level in [c.p, c.end): model_spec (merged) into *spec, and every entry of `result` - [off, off + len) of
// the record, in wire order over every occurrence of `result` - handed to on_entry(off, len).  Returns the status.  (The index
// kernel runs the same walk with a warp finding the entries of each result body: xr_warp_entries.)
template <class OnEntry>
B2_HD int xr_walk_response(Cursor& c, b200tfs_model_spec& spec, OnEntry& on_entry) {
  spec_reset(spec);
  uint32_t lo, hi;
#pragma unroll 1
  while (!c.err && xr_next_result(c, spec, &lo, &hi)) xr_entries(c, lo, hi, on_entry);
  return c.err;
}

// little-endian fixed32 at the cursor (4 bytes known to be there)
B2_HD uint32_t xr_fixed32(Cursor& c) {
  const uint32_t v = (uint32_t)rd8(c, c.p) | ((uint32_t)rd8(c, c.p + 1) << 8) | ((uint32_t)rd8(c, c.p + 2) << 16) |
                     ((uint32_t)rd8(c, c.p + 3) << 24);
  c.p += 4;
  return v;
}

// One Regression in [c.p, c.end): the float32 bits of `value` as the runtime returns it (0 when absent, signalling NaN quieted).
B2_HD uint32_t xr_regression(Cursor& c) {
  uint32_t v = 0;
#pragma unroll 1
  while (c.p < c.end && !c.err) {
    const uint32_t t = rd_tag(c);
    if (c.err) break;
    if (t == tag_of(1, WT_I32)) {
      if (c.end - c.p < 4) { c.err = B200TFS_E_PARSE; break; }
      v = xr_fixed32(c);
    } else skip_field(c, t);
  }
  return quiet_f32(v);
}

// One Classifications in [c.p, c.end): on_class(k, label_off, label_len, score bits) for its k-th Class, in wire order.
// Returns the class count.
template <class OnClass>
B2_HD uint32_t xr_classes(Cursor& c, OnClass& on_class) {
  uint32_t k = 0;
#pragma unroll 1
  while (c.p < c.end && !c.err) {
    const uint32_t t = rd_tag(c);
    if (c.err) break;
    if (t != tag_of(1, WT_LEN)) { skip_field(c, t); continue; }
    const uint32_t n = rd_len(c);
    if (c.err) break;
    const uint32_t outer = c.end;
    c.end = c.p + n;
    uint32_t lo = 0, ll = 0, score = 0;
#pragma unroll 1
    while (c.p < c.end && !c.err) {
      const uint32_t u = rd_tag(c);
      if (c.err) break;
      if (u == tag_of(1, WT_LEN)) {
        uint32_t len;
        const uint32_t at = rd_string(c, &len);
        if (c.err) break;
        lo = len ? at : 0; ll = len;
      } else if (u == tag_of(2, WT_I32)) {
        if (c.end - c.p < 4) { c.err = B200TFS_E_PARSE; break; }
        score = xr_fixed32(c);
      } else skip_field(c, u);
    }
    c.end = outer;
    if (c.err) break;
    on_class(k, lo, ll, quiet_f32(score));
    ++k;
  }
  return k;
}

}  // namespace b200tfs
