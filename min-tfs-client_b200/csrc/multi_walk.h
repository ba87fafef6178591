// multi_walk.h - the MultiInferenceResponse walk (inference.proto) that mi_index_kernel runs (multi_resp_kernels.cuh), built
// from walker.h's cursor helpers and example_walk.h's result walk.  The same source compiles for the host, where tests/native
// replays responses and mutants of them through it.
//
//   MultiInferenceResponse { repeated InferenceResult results = 1; }
//   InferenceResult { ModelSpec model_spec = 1; oneof result { ClassificationResult classification_result = 2;
//                                                              RegressionResult regression_result = 3; } }
//
// What the runtime does, and so what the walk does: every `results` field is its own InferenceResult; inside one, model_spec
// fields merge, a oneof member that occurs again merges (its entries concatenate), and a different member clears the one before
// it - whose bytes were parsed all the same, so a malformed cleared member is still a parse error.  Unknown fields and groups are
// skipped at every level; a known field with another wire type is an unknown field.
#pragma once
#include "example_walk.h"

namespace b200tfs {

constexpr uint32_t kMiClassify = 2, kMiRegress = 3;   // the oneof members' field numbers

// the member a task of kind B200TFS_RESP_* takes
B2_HD uint32_t mi_case_of(uint32_t kind) { return kind == B200TFS_RESP_CLASSIFY ? kMiClassify : kMiRegress; }

// The top level from c.p on, up to the next `results` field: other fields are skipped.  Returns true with the result's body in
// [*lo, *hi) (the cursor behind it), false at the end of the record or on an error.
B2_HD bool mi_next_result(Cursor& c, uint32_t* lo, uint32_t* hi) {
#pragma unroll 1
  while (c.p < c.end && !c.err) {
    const uint32_t tag = rd_tag(c);
    if (c.err) break;
    if (tag == tag_of(1, WT_LEN)) {
      const uint32_t m = rd_len(c);
      if (c.err) break;
      *lo = c.p; *hi = c.p + m;
      c.p += m;
      return true;
    }
    skip_field(c, tag);
  }
  return false;
}

// The next field of member `kase` in [c.p, c.end): true with its body in [*lo, *hi) (the cursor behind it).  Every other field is
// skipped.
B2_HD bool mi_next_member(Cursor& c, uint32_t kase, uint32_t* lo, uint32_t* hi) {
#pragma unroll 1
  while (c.p < c.end && !c.err) {
    const uint32_t tag = rd_tag(c);
    if (c.err) break;
    if (tag == tag_of(kase, WT_LEN)) {
      const uint32_t m = rd_len(c);
      if (c.err) break;
      *lo = c.p; *hi = c.p + m;
      c.p += m;
      return true;
    }
    skip_field(c, tag);
  }
  return false;
}

struct MiNoClass {
  B2_HD void operator()(uint32_t, uint32_t, uint32_t, uint32_t) {}
};
struct MiCheckEntry {   // every entry of a member body, walked to the end: what the runtime parses of a cleared member
  Cursor* c; uint32_t kase;
  B2_HD void operator()(uint32_t off, uint32_t len) {
    if (c->err) return;
    const uint32_t p0 = c->p, e0 = c->end;
    c->p = off; c->end = off + len;
    if (kase == kMiClassify) { MiNoClass s; xr_classes(*c, s); }
    else xr_regression(*c);
    c->p = p0; c->end = e0;
  }
};

// One InferenceResult body [lo, hi): its model_spec fields merged into *spec, the member that survives in *kase (0: none), and in
// *from where the run of that member starts - the tag of its first occurrence behind the last switch, so that from there on every
// member field is one of its occurrences.  Every member occurrence in front of *from was cleared: it is parsed to the end here.
// Leaves an error in c.err; the cursor's range is restored.
B2_HD void mi_result_case(Cursor& c, uint32_t lo, uint32_t hi, b200tfs_model_spec& spec, uint32_t* kase, uint32_t* from) {
  const uint32_t p0 = c.p, outer = c.end;
  uint32_t k = 0, f = lo;
  c.p = lo; c.end = hi;
#pragma unroll 1
  while (c.p < c.end && !c.err) {
    const uint32_t at = c.p, tag = rd_tag(c);
    if (c.err) break;
    if (tag == tag_of(1, WT_LEN)) {
      const uint32_t m = rd_len(c);
      if (c.err) break;
      const uint32_t e = c.end;
      c.end = c.p + m;
      walk_model_spec(c, spec);
      c.end = e;
    } else if (tag == tag_of(kMiClassify, WT_LEN) || tag == tag_of(kMiRegress, WT_LEN)) {
      const uint32_t m = rd_len(c);
      if (c.err) break;
      if (tag >> 3 != k) { k = tag >> 3; f = at; }
      c.p += m;
    } else skip_field(c, tag);
  }
  // the cleared members: every occurrence of either in front of the surviving run (none when f == lo)
#pragma unroll 1
  for (uint32_t m = kMiClassify; m <= kMiRegress && !c.err; ++m) {
    c.p = lo; c.end = f;
    uint32_t blo, bhi;
    MiCheckEntry chk{&c, m};
#pragma unroll 1
    while (!c.err && mi_next_member(c, m, &blo, &bhi)) xr_entries(c, blo, bhi, chk);
  }
  c.p = p0; c.end = outer;
  *kase = k; *from = f;
}

// Every entry of the run of member `kase` in [from, hi) parsed to the end: a result whose entries no task decodes (past the tasks,
// or not the member its task's method names) is still parsed by the runtime.  Leaves an error in c.err; the range is restored.
B2_HD void mi_check_run(Cursor& c, uint32_t kase, uint32_t from, uint32_t hi) {
  const uint32_t p0 = c.p, outer = c.end;
  c.p = from; c.end = hi;
  uint32_t blo, bhi;
  MiCheckEntry chk{&c, kase};
#pragma unroll 1
  while (!c.err && kase && mi_next_member(c, kase, &blo, &bhi)) xr_entries(c, blo, bhi, chk);
  c.p = p0; c.end = outer;
}

}  // namespace b200tfs
