// frame.h - deferred framing (plan.h): what frame_requests_kernel does for one request.  Host/device inline so that the host
// can run the very same code (b200tfs_request_frame_deferred: tests and bindings, no device needed).
//
// A request's program is looked at through a FrameView: its segments, values and terms (request-local indices), the value of
// every FT_TOTAL term already fetched, its slice of the blob.  On the device a warp stages all of that in shared memory with
// three rounds of parallel loads and one lane then runs frame_request_run out of shared memory - a lone lane chasing the
// tables through global memory paid ~60 dependent L2 round trips per request.
#pragma once
#include "plan.h"
#include "wire.h"

namespace b200tfs {

struct FrameView {
  const FrameSeg* segs;        // rq.n_seg
  const FrameVal* vals;        // rq.n_val; first_term is still the GLOBAL term index
  const FrameTerm* terms;      // the request's terms; term t of the request is global term rq.first_term + t
  const uint64_t* term_total;  // per request term: the job total of an FT_TOTAL term (others: unused)
  const uint8_t* blob;         // FS_BYTES offsets are global: blob[a - rq.first_blob]
  uint64_t* val;               // rq.n_val evaluated values (scratch)
};

// element e of a tiny packed-varint input, widened to 64 bits the way the protobuf runtime widens it (sign-extended if signed)
B2_HD uint64_t tiny_elem(const TinyVar& t, uint32_t e) {
  const uint8_t* p = t.src + (uint64_t)e * t.elem_size;
  uint64_t v = 0;
  for (uint32_t b = 0; b < t.elem_size; ++b) v |= (uint64_t)p[b] << (8 * b);
  if (t.is_signed && t.elem_size < 8 && (v >> (8 * t.elem_size - 1)) & 1) v |= ~0ull << (8 * t.elem_size);
  return v;
}
B2_HD uint64_t tiny_total(const TinyVar& t) {
  uint64_t s = 0;
  for (uint32_t e = 0; e < t.n; ++e) s += varint_len(tiny_elem(t, e));
  return s;
}

B2_HD uint64_t frame_seg_len(const FrameSeg& sg, const uint64_t* val) {
  switch (sg.kind) {
    case FS_BYTES: return sg.b;
    case FS_VARINT: return varint_len(val[sg.a]);
    case FS_BE32: return 4;
    case FS_ITEM: case FS_SMALL: return sg.b;      // the host wrote the payload's length next to its index
    default: return val[sg.b];                     // FS_VARJOB / FS_TINYVAR: b = the value that is its packed length
  }
}

B2_HD void frame_request_run(const FrameTables& ft, const FrameReq& rq, const FrameView& V, uint32_t r) {
  uint64_t* val = V.val;
  for (uint32_t v = 0; v < rq.n_val; ++v) {
    const FrameVal fv = V.vals[v];
    uint64_t x = (uint64_t)fv.c;
    for (uint32_t k = 0; k < fv.n_terms; ++k) {
      const uint32_t ti = fv.first_term - rq.first_term + k;
      const FrameTerm t = V.terms[ti];
      if (t.kind == FT_TOTAL || t.kind == FT_TINY) x += V.term_total[ti];
      else if (t.kind == FT_VAL) x += val[t.idx];
      else x += varint_len(val[t.idx]);
    }
    val[v] = x;
  }
  uint64_t pad = 0;
  if (rq.align_seg != ~0u) {
    uint64_t before = 0;
    for (uint32_t k = 0; k < rq.align_seg; ++k) before += frame_seg_len(V.segs[k], val);
    pad = (128 - ((rq.slot_off + before) & 127)) & 127;
  }
  const uint64_t total = val[rq.total_val];
  uint64_t start = rq.slot_off + pad;
  if (rq.anchor_seg != ~0u) {     // the host fixed where the payload goes: the record starts as far in front of it as its prefix is long
    uint64_t before = 0;
    for (uint32_t k = 0; k < rq.anchor_seg; ++k) before += frame_seg_len(V.segs[k], val);
    start = rq.anchor_off - before;     // >= slot_off: the host put the anchor behind the longest prefix possible
    pad = start - rq.slot_off;
  }
  ft.rec_off[r] = start; ft.rec_len[r] = total;
  if (pad + total > rq.slot_cap || total > 0x7FFFFFFFull + 5) {   // cannot happen with the host's worst-case slots; never write outside one
    ft.status[r] = total > 0x7FFFFFFFull + 5 ? B200TFS_E_TOOBIG : B200TFS_E_SIZE;
    for (uint32_t k = 0; k < rq.n_seg; ++k) {   // park the movers on an empty range
      const FrameSeg sg = V.segs[k];
      if (sg.kind == FS_ITEM) ft.items[sg.a].n_out = 0;
      else if (sg.kind == FS_SMALL) ft.smalls[sg.a].n_out = 0;
      else if (sg.kind == FS_VARJOB) { ft.jobs[sg.a].dst = ft.arena + rq.slot_off; ft.jobs[sg.a].cap = 0; }   // (FS_TINYVAR: nothing runs behind it)
    }
    return;
  }
  ft.status[r] = B200TFS_OK;
  uint8_t* w = ft.arena + start;
  for (uint32_t k = 0; k < rq.n_seg; ++k) {
    const FrameSeg sg = V.segs[k];
    switch (sg.kind) {
      case FS_BYTES: { const uint8_t* b = V.blob + (sg.a - rq.first_blob); for (uint32_t q = 0; q < sg.b; ++q) w[q] = b[q]; w += sg.b; break; }
      case FS_VARINT: w += put_varint(w, val[sg.a]); break;
      case FS_BE32: { const uint64_t m = val[sg.a]; w[0] = (uint8_t)(m >> 24); w[1] = (uint8_t)(m >> 16); w[2] = (uint8_t)(m >> 8); w[3] = (uint8_t)m; w += 4; break; }
      case FS_ITEM: ft.items[sg.a].dst = w; w += sg.b; break;
      case FS_SMALL: ft.smalls[sg.a].dst = w; w += sg.b; break;
      case FS_TINYVAR: { const TinyVar t = ft.tiny[sg.a]; for (uint32_t e = 0; e < t.n; ++e) w += put_varint(w, tiny_elem(t, e)); break; }
      default: { const uint64_t L = val[sg.b]; ft.jobs[sg.a].dst = w; ft.jobs[sg.a].cap = L; w += L; break; }
    }
  }
}

// straight from the tables (host; device fallback for a request too large for the shared-memory staging): FT_TOTAL terms are
// fetched into ft.scratch_terms first
B2_HD void frame_request(const FrameTables& ft, uint32_t r) {
  const FrameReq rq = ft.reqs[r];
  uint64_t* tt = ft.scratch_terms + rq.first_term;
  for (uint32_t t = 0; t < rq.n_term; ++t) {
    const FrameTerm ft_t = ft.terms[rq.first_term + t];
    tt[t] = ft_t.kind == FT_TOTAL ? (uint64_t)ft.totals[ft_t.idx] : ft_t.kind == FT_TINY ? tiny_total(ft.tiny[ft_t.idx]) : 0;
  }
  FrameView V{ft.segs + rq.first_seg, ft.vals + rq.first_val, ft.terms + rq.first_term, tt, ft.blob + rq.first_blob, ft.scratch_vals + rq.first_val};
  frame_request_run(ft, rq, V, r);
}

}  // namespace b200tfs
