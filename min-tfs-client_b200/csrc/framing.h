// framing.h - the PredictRequest framing writers: model_spec, a map entry's header, a TensorProto's header.  Host/device inline
// and templated on where the bytes go (`Out`: byte / varint / bytes), so that the host planner (codec_host.cpp), the padded
// encode's host emulation and its framing kernel (unpad.h) all write framing through this one copy of the protobuf rules.
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
  uint64_t payload_len = 0;  // bytes of the values field body on the wire (0: field omitted, or not known yet: unmeasured)
  uint64_t header_len = 0;   // bytes before the payload
  uint32_t op = OP_COPY;     // MoveOp for fixed-width payloads
  bool varint = false;       // payload produced by the varint kernels
  bool unmeasured = false;   // a packed-varint payload the deferred encode counts on the device: the header ends at the values
                             // tag, and the length behind it is the framing kernel's to write
  uint32_t field = 0;        // field number the values go into
  uint64_t shape_len = 0;    // bytes of the TensorShapeProto body
  DtypeInfo src_info{}, wire_info{};
};

// Where the framing writers below put their bytes: raw stores at `w` (the immediate planner writes the blob in place; the padded
// encode writes the record), a CountOut that only counts them, or a DeferredBuilder (varint_host.inc), which also takes Pending
// lengths - values its framing program computes on the device
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

// model_spec{ 0A vi name [12 vi {08 vi(version)}] } of a PredictRequest or a tf.Example request
struct SpecLayout {
  uint64_t body = 0, version_len = 0;
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
}

// a map entry's header: 12 vi(entry_len) 0A vi(key_len) key 12 vi(tp_len)
template <class Out, class Len>
B2_HD void write_entry_header(Out& o, const b200tfs_tensor& t, Len entry_len, Len tp_len) {
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
// [tag vi(payload_len)] - an unmeasured payload's tag without its length; nothing for a pre-serialised TensorProto
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
  if (L.payload_len || L.unmeasured) o.varint(tag_of(L.field, WT_LEN));
  if (L.payload_len) o.varint(L.payload_len);
}

}  // namespace b200tfs
