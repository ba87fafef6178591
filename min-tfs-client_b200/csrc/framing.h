// framing.h - the PredictRequest framing writers: model_spec, a map entry's header, a TensorProto's header and the request loop
// around them.  Host/device inline and templated on where the bytes go (`Out`: byte / varint / bytes), so that the host planner
// (codec_host.cpp), the deferred encode (frame_requests_kernel and its host emulation) and the padded encode (unpad.h) all write
// framing through this one copy of the protobuf rules.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include "../../include/b200tfs.h"
#include "plan.h"
#include "wire.h"

namespace b200tfs {

struct TensorLayout {
  uint64_t n_elems = 0;
  uint64_t payload_len = 0;  // bytes of the values field body on the wire (0: field omitted, or counted on the device later)
  uint64_t header_len = 0;   // bytes before the payload
  uint32_t op = OP_COPY;     // MoveOp for fixed-width payloads
  bool varint = false;       // payload produced by the varint kernels
  uint32_t field = 0;        // field number the values go into; F_STRING: repeated string_val, each value its own 42 vi(len)
                             // bytes field, so the payload (all of them) has no enclosing tag and length
  uint64_t shape_len = 0;    // bytes of the TensorShapeProto body
  DtypeInfo src_info{}, wire_info{};
};

// Where the framing writers below put their bytes: raw stores at `w` (the immediate planner writes the blob in place; the framing
// kernels write the record), or a CountOut that only counts them
struct RawOut {
  uint8_t* w;
  B2_HD void byte(uint8_t b) { *w++ = b; }
  B2_HD void varint(uint64_t v) { w += put_varint(w, v); }
  B2_HD void bytes(const void* p, size_t n) {
#if defined(__CUDA_ARCH__)
    const uint8_t* s = (const uint8_t*)p;
    for (size_t i = 0; i < n; ++i) w[i] = s[i];
    w += n;
#else
    if (n) { memcpy(w, p, n); w += n; }
#endif
  }
  B2_HD void skip(uint64_t n) { w += n; }
  B2_HD uint64_t pos() const { return (uint64_t)(uintptr_t)w; }
};
struct CountOut {
  uint64_t n = 0;
  B2_HD void byte(uint8_t) { n += 1; }
  B2_HD void varint(uint64_t v) { n += varint_len(v); }
  B2_HD void bytes(const void*, size_t k) { n += k; }
  B2_HD void skip(uint64_t k) { n += k; }
  B2_HD uint64_t pos() const { return n; }
};

// model_spec{ 0A vi name [12 vi {08 vi(version)}] [1A vi signature_name] [22 vi version_label] } of a PredictRequest or a
// tf.Example request, in field-number order.  signature_name is a proto3 scalar (empty: not written); version_label is a member
// of the version_choice oneof, so a set label is written even when empty (22 00).  The strings are host memory: the spec is
// written on the host and copied as bytes by every kernel that places it.
struct SpecLayout {
  uint64_t body = 0, version_len = 0;
  const char* sig = nullptr; uint64_t sig_len = 0;
  const char* label = nullptr; int64_t label_len = -1;   // < 0: no version_label
  B2_HD uint64_t field() const { return 1 + varint_len(body) + body; }   // with its tag and length
};

template <class Out, class Req>
B2_HD void write_model_spec(Out& o, const Req& r, const SpecLayout& S) {
  o.byte(0x0A); o.varint(S.body);
  if (r.model_name_len) { o.byte(0x0A); o.varint((uint64_t)r.model_name_len); o.bytes(r.model_name, (size_t)r.model_name_len); }
  if (r.has_version) {
    o.byte(0x12); o.byte((uint8_t)S.version_len);
    if (r.version) { o.byte(0x08); o.varint((uint64_t)r.version); }
  }
  if (S.sig_len) { o.byte(0x1A); o.varint(S.sig_len); o.bytes(S.sig, (size_t)S.sig_len); }
  if (S.label_len >= 0) { o.byte(0x22); o.varint((uint64_t)S.label_len); o.bytes(S.label, (size_t)S.label_len); }
}

// PredictRequest.output_filter: {1A vi(len) name}* in the order given (no sorting, no de-duplication), behind the last inputs
// entry.  Host only, like the spec: the deferred and padded encodes copy these bytes from their blob.
template <class Out>
void write_output_filter(Out& o, const b200tfs_request_spec* s) {
  for (int64_t i = 0; s && i < s->n_output_filter; ++i) {
    o.byte(0x1A); o.varint((uint64_t)s->output_filter_len[i]); o.bytes(s->output_filter[i], (size_t)s->output_filter_len[i]);
  }
}

// a map entry's header: 12 vi(entry_len) 0A vi(key_len) key 12 vi(tp_len)
template <class Out>
B2_HD void write_entry_header(Out& o, const b200tfs_tensor& t, uint64_t entry_len, uint64_t tp_len) {
  o.byte(0x12); o.varint(entry_len);
  o.byte(0x0A); o.varint((uint64_t)t.key_len); o.bytes(t.key, (size_t)t.key_len);
  o.byte(0x12); o.varint(tp_len);
}

// bytes of the TensorShapeProto body: one Dim per axis, Dim(size=0) empty (Q2)
B2_HD uint64_t shape_body_len(int32_t rank, const int64_t* dims) {
  uint64_t s = 0;
  for (int i = 0; i < rank; ++i) s += 2 + (dims[i] ? 1 + varint_len((uint64_t)dims[i]) : 0);
  return s;
}

// the header_len bytes in front of a tensor's payload: 08 vi(dtype) 12 vi(shape_len) {12 vi(dim_len) [08 vi(size)]}*
// [tag vi(payload_len)] (not for string_val, whose values carry their own tags); nothing for a pre-serialised TensorProto
template <class Out>
B2_HD void write_tensor_header(Out& o, const b200tfs_tensor& t, const TensorLayout& L) {
  if (t.flags & B200TFS_F_PRESERIALIZED) return;
  o.byte(0x08); o.varint((uint64_t)(uint32_t)t.wire_dtype);
  o.byte(0x12); o.varint(L.shape_len);
  for (int i = 0; i < t.rank; ++i) {
    const uint64_t d = (uint64_t)t.dims[i];
    o.byte(0x12);
    if (d) { o.byte((uint8_t)(1 + varint_len(d))); o.byte(0x08); o.varint(d); }
    else o.byte(0x00);  // Dim(size=0) is an empty sub-message (Q2)
  }
  if (L.payload_len && L.field != F_STRING) { o.varint(tag_of(L.field, WT_LEN)); o.varint(L.payload_len); }
}

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

// The framing of one PredictRequest through `o`: [00 be32(msg)] model_spec {entry header, tensor header, payload}* output_filter.
// `Req` supplies what differs between the callers: spec(o) writes the model_spec field, input(j, t, L) fills in input j of the
// wire order (key, dims, wire dtype, flags; field, payload_len), payload(o, j, t, L) writes, skips or records its payload_len
// bytes and tail(o) writes the output_filter run.
template <class Out, class Req>
B2_HD void write_request(Out& o, Req& q, uint32_t n_in, bool grpc, uint64_t msg) {
  if (grpc) { o.byte(0); o.byte((uint8_t)(msg >> 24)); o.byte((uint8_t)(msg >> 16)); o.byte((uint8_t)(msg >> 8)); o.byte((uint8_t)msg); }
  q.spec(o);
  for (uint32_t j = 0; j < n_in; ++j) {
    b200tfs_tensor t{};
    TensorLayout L;
    q.input(j, t, L);
    CountOut h;
    write_tensor_header(h, t, L);
    const uint64_t tp = h.n + L.payload_len;
    const uint64_t el = 1 + varint_len((uint64_t)t.key_len) + (uint64_t)t.key_len + 1 + varint_len(tp) + tp;
    write_entry_header(o, t, el, tp);
    write_tensor_header(o, t, L);
    q.payload(o, j, t, L);
  }
  q.tail(o);
}

// ---- the deferred encode (plan.h "deferred framing") ----------------------------------------------------------------------
// write_request's view of one request of a deferred encode.  Payload lengths are read as the framing is written: a varint job's
// from the counting kernel's totals, a tiny input's by counting it, a fixed one's from the table.
struct DeferredRequest {
  const FrameTables& ft;
  const DeferredReq& q;
  uint64_t* payload_off;           // write pass (may be null): where each input's payload landed in the arena, and its length
  uint64_t* payload_len;
  DeferredIn in{};                 // the input input() read last
  uint64_t align_at = 0;           // count pass: where input q.align_in's payload starts, from the record's first byte
  template <class Out> B2_HD void spec(Out& o) { o.bytes(ft.blob + q.spec_off, q.spec_len); }
  template <class Out> B2_HD void tail(Out& o) { o.bytes(ft.blob + q.spec_off + q.spec_len, q.tail_len); }
  B2_HD void input(uint32_t j, b200tfs_tensor& t, TensorLayout& L) {
    in = ft.ins[q.first_in + j];
    t.key = (const char*)ft.blob + in.key_off; t.key_len = in.key_len;
    t.dims = (const int64_t*)(ft.blob + in.dims_off); t.rank = in.rank;
    t.wire_dtype = in.wire_dtype; t.flags = in.flags;
    L.field = in.field;
    L.shape_len = shape_body_len(in.rank, t.dims);
    L.payload_len = in.kind == DP_JOB ? (uint64_t)ft.totals[in.idx] : in.kind == DP_TINY ? tiny_total(ft.tiny[in.idx]) : in.len;
  }
  B2_HD void payload(CountOut& o, uint32_t j, const b200tfs_tensor&, const TensorLayout& L) {
    if (j == q.align_in) align_at = o.n;
    o.skip(L.payload_len);
  }
  B2_HD void payload(RawOut& o, uint32_t j, const b200tfs_tensor&, const TensorLayout& L) {
    if (payload_off && in.kind != DP_NONE) { payload_off[j] = (uint64_t)(o.w - ft.arena); payload_len[j] = L.payload_len; }
    switch (in.kind) {
      case DP_ITEM: ft.items[in.idx].dst = o.w; break;
      case DP_SMALL: ft.smalls[in.idx].dst = o.w; break;
      case DP_JOB: ft.jobs[in.idx].dst = o.w; ft.jobs[in.idx].cap = L.payload_len; break;
      case DP_TINY: {
        const TinyVar tv = ft.tiny[in.idx];
        for (uint32_t e = 0; e < tv.n; ++e) o.varint(tiny_elem(tv, e));
        return;
      }
      default: break;
    }
    o.skip(L.payload_len);
  }
};

// Request r of a deferred encode: counted, placed in its slot (its align input's payload 128-byte aligned, like the host planner's
// place_record, or around its anchor), checked, then written - all of frame_requests_kernel's work for it, and what
// b200tfs_request_frame_deferred runs on the host.  payload_off / payload_len (may be null) receive, per input of the wire order
// that has a payload, where it landed in the arena and its length.
B2_HD void frame_request(const FrameTables& ft, uint32_t r, uint64_t* payload_off = nullptr, uint64_t* payload_len = nullptr) {
  const DeferredReq q = ft.reqs[r];
  DeferredRequest D{ft, q, payload_off, payload_len};
  CountOut c;
  write_request(c, D, q.n_in, q.grpc != 0, 0);     // the prefix's length does not depend on its value
  const uint64_t total = c.n;
  uint64_t pad = 0;
  if (q.align_in != ~0u) pad = (128 - ((q.slot_off + D.align_at) & 127)) & 127;
  uint64_t start = q.slot_off + pad;
  if (q.anchor_in != ~0u) {     // the host fixed where the payload (the align input's) goes: the record starts as far in front of
    start = q.anchor_off - D.align_at;     // it as its prefix is long; >= slot_off: the host put the anchor behind the longest prefix possible
    pad = start - q.slot_off;
  }
  ft.rec_off[r] = start; ft.rec_len[r] = total;
  if (pad + total > q.slot_cap || total > 0x7FFFFFFFull + 5) {   // cannot happen with the host's worst-case slots; never write outside one
    ft.status[r] = total > 0x7FFFFFFFull + 5 ? B200TFS_E_TOOBIG : B200TFS_E_SIZE;
    for (uint32_t j = 0; j < q.n_in; ++j) {   // park the movers on an empty range
      const DeferredIn in = ft.ins[q.first_in + j];
      if (in.kind == DP_ITEM) ft.items[in.idx].n_out = 0;
      else if (in.kind == DP_SMALL) ft.smalls[in.idx].n_out = 0;
      else if (in.kind == DP_JOB) { ft.jobs[in.idx].dst = ft.arena + q.slot_off; ft.jobs[in.idx].cap = 0; }   // (DP_TINY: nothing runs behind it)
    }
    return;
  }
  ft.status[r] = B200TFS_OK;
  RawOut o{ft.arena + start};
  write_request(o, D, q.n_in, q.grpc != 0, total - (q.grpc ? 5 : 0));
}

}  // namespace b200tfs
