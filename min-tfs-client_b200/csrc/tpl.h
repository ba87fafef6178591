// tpl.h - the framing template of the single-launch decode, shared by the kernel (kernels.cu: the CTA of record 0
// learns it while walking) and the host (codec_host.cpp: when the wire is in host memory - it always is behind the gRPC
// response_deserializer, prediction_service_pb2_grpc.py:53 - the library walks record 0 itself before the launch, so that
// even the first launch takes the template path).  Everything here is host/device inline; no allocation.
//
// A template is: the record's framing bytes (everything that is not a value chunk), where the value chunks lie, where
// each goes in the destination slot, and the finished table.  A record with the same length and the same framing bytes at
// the same positions parses identically, so its CTAs take their tiles straight from the template.
#pragma once
#include "plan.h"
#include "walker.h"
#include "wire.h"

namespace b200tfs {

B2_HD uint32_t tpl_tiles_for(uint64_t n_out, uint32_t vpt) {
  const uint64_t vecs = (n_out + 15) >> 4;
  const uint64_t t = (vecs + vpt - 1) / vpt;
  return t ? (uint32_t)t : 1u;
}

// Destination layout of a walked record: every fixed-width output that decoded cleanly gets a 256-byte aligned range of
// the record's slot, in table order.  Returns the bytes of the slot in use.  (String outputs are tabulated only; so are
// varint outputs unless `varints` != 0 - b200tfs_set_decode_varints - which gives them ranges in the same order.)
// `cast` != 0: DT_FLOAT outputs leave as DT_HALF / DT_BFLOAT16 (two bytes per element; dst_bytes says so, dtype stays the wire's).
B2_HD bool tpl_narrows(uint32_t cast, int32_t dtype) { return cast != 0 && dtype == DT_FLOAT; }
B2_HD uint32_t tpl_move_op(uint32_t cast, int32_t dtype) {
  if (dtype != DT_FLOAT) return OP_COPY;
  return cast == (uint32_t)DT_HALF ? OP_F2H : cast == (uint32_t)DT_BFLOAT16 ? OP_F2B : OP_QUIET_DST;
}
B2_HD bool tpl_gets_range(uint32_t varints, int32_t dtype) {
  const uint32_t kind = dtype_info(dtype).kind;
  return kind == VK_FIXED || (varints && (kind == VK_VARINT || kind == VK_BOOL));
}
B2_HD uint64_t tpl_layout_outputs(b200tfs_output* outs, int cnt, uint64_t dst_stride, uint32_t cast = 0, uint32_t varints = 0) {
  uint64_t cursor = 0;
  for (int k = 0; k < cnt; ++k) {
    b200tfs_output& o = outs[k];
    if (o.status != B200TFS_OK || !o.n_elems) continue;
    if (!tpl_gets_range(varints, o.dtype)) continue;
    if (tpl_narrows(cast, o.dtype)) o.dst_bytes = o.n_elems * 2;
    cursor = (cursor + 255) & ~255ull;
    if (cursor + o.dst_bytes > dst_stride) { o.status = B200TFS_E_SIZE; continue; }
    o.dst_off = cursor;
    cursor += o.dst_bytes;
  }
  return cursor;
}

// Build the template of a walked record (chunks sorted by wire offset, framing bytes).  T->in.head.valid stays 0 when the
// record does not qualify.  `c` is the cursor the record was walked with (its bytes are read through rd8).
B2_HD void tpl_learn(Template* T, Cursor& c, uint32_t len, const b200tfs_output* outs, int cnt, const b200tfs_model_spec& spec,
                     int st, uint32_t vpt, uint64_t dst_need, uint32_t serial, uint32_t cast = 0, uint32_t varints = 0) {
  T->in.head.valid = 0;
  if (st != B200TFS_OK || cnt > kFusedMaxOutputs) return;
  TplChunk ch[kTplChunks];
  uint32_t n = 0;
  for (int k = 0; k < cnt; ++k) {
    const b200tfs_output& o = outs[k];
    if (o.status != B200TFS_OK && o.status != B200TFS_E_SHAPE && o.status != B200TFS_E_KEY) return;
    const DtypeInfo di = dtype_info(o.dtype);
    const bool moved = (o.status == B200TFS_OK) && di.kind == VK_FIXED && o.n_elems;
    // A template stands for "identical framing bytes parse identically" with every value chunk opaque.  That holds for packed
    // occurrences (length-delimited); an UNPACKED varint element's own continuation bits decide where the next tag starts, so
    // a record with unpacked elements is never learnt (it takes the walk every time), nor is one whose runs are strided / spilled.
    if (o.flags & (B200TFS_OF_UNPACKED | B200TFS_OF_SPILLED)) return;
    uint32_t run = 0;
    for (int q = 0; q < o.n_runs; ++q) {
      if (n >= kTplChunks || o.runs[q].count != 1) return;
      TplChunk x;
      x.wire_off = (uint32_t)o.runs[q].off; x.len = o.runs[q].len;
      const bool narrow = tpl_narrows(cast, o.dtype);      // run lengths of a float field are multiples of 4 (else the walk failed)
      x.dst_off = (uint32_t)o.dst_off + (narrow ? run / 2 : run); x.op = tpl_move_op(cast, o.dtype);
      x.n_tiles = moved ? tpl_tiles_for(narrow ? o.runs[q].len / 2 : o.runs[q].len, vpt) : 0u;
      x.is_varint = (o.flags & B200TFS_OF_VARINT) ? 1u : 0u; x.fpos = 0; x.pad = 0;
      if (o.dst_off + run + o.runs[q].len > 0xFFFFFFFFull) return;
      run += o.runs[q].len;
      ch[n++] = x;
    }
    if (o.content_len) {  // tensor_content: opaque like a payload, never moved here
      if (n >= kTplChunks) return;
      TplChunk x;
      x.wire_off = (uint32_t)o.content_off; x.len = (uint32_t)o.content_len; x.dst_off = 0; x.op = OP_COPY; x.n_tiles = 0;
      x.is_varint = 0; x.fpos = 0; x.pad = 0;
      ch[n++] = x;
    }
  }
  for (uint32_t i = 1; i < n; ++i) {  // by wire offset; tiles are handed out in this order
    TplChunk x = ch[i];
    uint32_t k = i;
    while (k > 0 && ch[k - 1].wire_off > x.wire_off) { ch[k] = ch[k - 1]; --k; }
    ch[k] = x;
  }
  uint32_t payload = 0, tiles = 0;
  for (uint32_t i = 0; i < n; ++i) {
    if (i && ch[i].wire_off < ch[i - 1].wire_off + ch[i - 1].len) return;  // overlapping: never, but be safe
    ch[i].fpos = ch[i].wire_off - payload;
    payload += ch[i].len;
    tiles += ch[i].n_tiles;
  }
  const uint32_t framing = len - payload;
  if (framing > kTplFraming) return;
  uint32_t w = 0, ci = 0;
  for (uint32_t i = 0; i < framing; ++i) {
    while (ci < n && ch[ci].wire_off == w) { w += ch[ci].len; ++ci; }
    T->in.framing[i] = rd8(c, w++);
  }
  for (uint32_t i = framing; i < kTplFraming; ++i) T->in.framing[i] = 0;
  for (uint32_t i = 0; i < kTplChunks; ++i) {
    if (i < n) T->in.chunk[i] = ch[i];
    else { TplChunk z; z.wire_off = z.len = z.dst_off = z.op = z.n_tiles = z.is_varint = z.fpos = z.pad = 0; T->in.chunk[i] = z; }
  }
  TplHead& h = T->in.head;
  h.n_chunks = n; h.n_outs = (uint32_t)cnt; h.framing_len = framing; h.rec_len = len; h.vpt = vpt; h.total_tiles = tiles;
  h.dst_need = dst_need; h.serial = serial; h.cast = cast; h.varints = varints; h.pad = 0;
  T->spec = spec;
  for (int k = 0; k < cnt; ++k) T->outs[k] = outs[k];
  h.valid = 1;   // device callers fence before publishing the structure to other CTAs / launches
}

}  // namespace b200tfs
