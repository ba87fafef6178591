// example_kernels.cuh - Classify / Regress requests: a batch of tf.Examples from columnar arrays (plan.h ExTables; planned by
// example_host.inc).  Included by kernels.cu inside namespace b200tfs, after concat_scan.
//
//   ex_count_kernel  requests whose size depends on their values (an integer or a ragged column): one warp per example finds
//                    the packed length of every integer row, then the example's byte length through its nested lengths (list <-
//                    Feature <- map entry <- Features <- Example); one CTA per kExTile examples leaves their sum in tile_sum
//   ex_scan_kernel   the same tiles: the tile's offset is the sum of the tiles before it in its request (read, never waited
//                    for: the count kernel has finished), then a block scan of the example sizes gives every example's offset
//   ex_emit_kernel   one CTA per contiguous range of examples, i.e. of wire: warps write whole examples (framing, converted float
//                    rows, int64 varints) into a shared-memory image of the wire, which the CTA stores with aligned 128-bit
//                    vectors; an example larger than the image is written in place by one warp.  ex_emit_predict_kernel is the
//                    same for the spans of Predict requests, whose examples start with the string_val tag
//   ex_frame_kernel  one warp per request: the examples' total, the request prefix in front of the anchor (an example_list or
//                    a Predict string_val, plan.h ExReq), rec_off / rec_len / status to pinned memory.  A call with contexts
//                    (ExampleListWithContext, plan.h ExCtxRef) runs ex_frame_context_kernel instead, whose warp also writes its
//                    request's context behind the examples; count and scan size the contexts as one-example entries
//   ex_seq_count_kernel, ex_emit_sequence_kernel   SequenceExample requests (plan.h sq_*), only in a call that has one: their
//                    tiles and spans follow all the others; the scan and frame kernels take them as they take examples
//
// count, emit and the example writer take an ExMode: a call with a bytes column launches the kExColumns instantiations, a call
// with a ragged numeric column (and none of bytes) the kExRagged ones, in which a ragged column's row ends after ex_elems
// elements; every other call runs the kExDense ones, which read row_elems as before.  kExColumns takes ragged rows too, and
// bytes rows: a row's strings are cut from one byte buffer by int64 offsets (ex_str_ends), one string per lane.
//
// What the reference does here: requests.py examples_from_input_dict (a Python loop per example and per feature) and the
// protobuf runtime serialising the ClassificationRequest / RegressionRequest it filled, or every example and then the
// PredictRequest whose DT_STRING input holds them.

// float32 bits of element j of a float row: what astype(float32) and the trip through a Python float give
__device__ __forceinline__ uint32_t ex_f64_to_f32_bits(uint64_t d) {
  if ((d & 0x7FFFFFFFFFFFFFFFull) > 0x7FF0000000000000ull)      // NaN: quieted, the top 22 payload bits kept (x86 cvtsd2ss)
    return ((uint32_t)(d >> 32) & 0x80000000u) | 0x7FC00000u | (uint32_t)((d & 0x000FFFFFFFFFFFFFull) >> 29);
  return __float_as_uint(__double2float_rn(__longlong_as_double((long long)d)));
}
__device__ __forceinline__ uint32_t ex_float_bits(const ExFeat& f, const uint8_t* row, uint64_t j) {
  if (f.op == EXO_F32) return quiet_f32(*reinterpret_cast<const uint32_t*>(row + 4 * j));
  if (f.op == EXO_F64) return ex_f64_to_f32_bits(*reinterpret_cast<const unsigned long long*>(row + 8 * j));
  return widen_f16(*reinterpret_cast<const uint16_t*>(row + 2 * j));
}
// element of an integer row as astype(int64) gives it (bool: any nonzero byte is 1)
__device__ __forceinline__ uint64_t ex_int(const ExFeat& f, const uint8_t* p) {
  switch (f.esz) {
    case 1: { const uint8_t t = *p; return f.op == EXO_BOOL ? (uint64_t)(t != 0) : f.sgn ? (uint64_t)(int64_t)(int8_t)t : t; }
    case 2: { const uint16_t t = *reinterpret_cast<const uint16_t*>(p); return f.sgn ? (uint64_t)(int64_t)(int16_t)t : t; }
    case 4: { const uint32_t t = *reinterpret_cast<const uint32_t*>(p); return f.sgn ? (uint64_t)(int64_t)(int32_t)t : t; }
    default: return *reinterpret_cast<const unsigned long long*>(p);
  }
}
// elements of example i's row: a ragged column's length, clamped to [0, max_len] (the count kernel flags one that was not), in
// steps of `unit`; row_elems for a dense column
template <int kMode>
__device__ __forceinline__ uint64_t ex_elems(const ExFeat& f, uint64_t i) {
  if (kMode == kExDense || !f.lengths) return f.row_elems;
  const int64_t l = f.lengths[i];
  return (l < 0 ? 0ull : min((uint64_t)l, f.max_len)) * f.unit;
}
template <int kMode>
__device__ __forceinline__ uint64_t ex_payload(const ExTables& T, const ExReq& q, const ExFeat& f, uint64_t i) {
  return f.op < EXO_INT ? 4 * ex_elems<kMode>(f, i) : T.L[q.L0 + i * q.n_int + f.lcol];
}
// the map entry of a feature whose list payload is P bytes
template <int kMode>
__device__ __forceinline__ uint64_t ex_feat_entry_len(const ExFeat& f, uint64_t P, uint64_t* hl) {
  return kMode == kExColumns && f.op == EXO_BYTES ? ex_bytes_entry_len(P, f.key_len, hl) : ex_entry_len(P, f.key_len, hl);
}
__device__ __forceinline__ uint64_t warp_sum64(uint64_t v) {
#pragma unroll
  for (int d = 16; d; d >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, d);
  return v;
}
// the sum of v over this lane and the lanes below it
__device__ __forceinline__ uint64_t warp_incl_scan64(uint64_t v) {
  const uint32_t lane = threadIdx.x & 31;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint64_t y = __shfl_up_sync(0xFFFFFFFFu, v, d);
    if (lane >= (uint32_t)d) v += y;
  }
  return v;
}

// ---- bytes rows ----
// Example i's row of a bytes column is strings b .. b + ne of the column (b = i * row_stride), and the kernels read offsets
// o[b .. b + ne] and o[b + row_elems], the next row's start.  A valid row has 0 <= o[b] <= ... <= o[b + ne] <= o[b + row_elems]
// <= data_len, so the rows of a valid request are disjoint and in order.  Count and emit both see the offsets through
// ex_str_ends: the row is clamped to [lo, hi] = [o[b], o[b + row_elems]] clamped into [0, data_len] (hi >= lo, and at most 4 GiB
// past lo: no request under 2 GiB has a longer row), and every offset into [lo, hi] with a running maximum.  So both kernels
// agree on every length, whatever the offsets hold, and no read leaves [data, data + data_len).
__device__ __forceinline__ uint64_t ex_clamp_off(int64_t v, uint64_t lo, uint64_t hi) {
  return v < 0 ? lo : min(max((uint64_t)v, lo), hi);
}
__device__ __forceinline__ void ex_row_bounds(const ExFeat& f, uint64_t b, uint64_t* lo, uint64_t* hi) {
  *lo = ex_clamp_off(f.offsets[b], 0, f.data_len);
  *hi = min(ex_clamp_off(f.offsets[b + f.row_elems], *lo, f.data_len), *lo + ((uint64_t)1 << 32));
}
// Warp-collective, over strings j0 .. j0 + 31 of a row (lane: string j0 + lane, < ne): the end of the lane's string, and through
// *start its start; *carry (the end of string j0 - 1, lo for j0 = 0) moves on to the end of string j0 + 31.
__device__ __forceinline__ uint64_t ex_str_ends(const ExFeat& f, uint64_t b, uint64_t ne, uint64_t j0, uint64_t lo, uint64_t hi,
                                                uint64_t* carry, uint64_t* start) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t j = j0 + lane;
  uint64_t e = j < ne ? ex_clamp_off(f.offsets[b + j + 1], lo, hi) : hi;
  e = max(e, *carry);
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint64_t x = __shfl_up_sync(0xFFFFFFFFu, e, d);
    if (lane >= (uint32_t)d) e = max(e, x);
  }
  const uint64_t s = __shfl_up_sync(0xFFFFFFFFu, e, 1);
  *start = lane ? s : *carry;
  *carry = __shfl_sync(0xFFFFFFFFu, e, 31);
  return e;
}
// Example i's bytes row at d, its list payload (L) already known: the {0A vi(len) bytes} field of every string.
__device__ __forceinline__ void ex_write_bytes(const ExFeat& f, uint64_t i, uint64_t ne, uint8_t* d) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t b = i * f.row_stride;
  uint64_t lo, hi, carry, base = 0;
  ex_row_bounds(f, b, &lo, &hi);
  carry = lo;
  for (uint64_t j0 = 0; j0 < ne; j0 += 32) {
    uint64_t s;
    const uint64_t e = ex_str_ends(f, b, ne, j0, lo, hi, &carry, &s);
    const uint64_t len = j0 + lane < ne ? e - s : 0;
    const uint64_t sz = j0 + lane < ne ? string_value_len(len) : 0;
    uint64_t incl = sz;
#pragma unroll
    for (int dd = 1; dd < 32; dd <<= 1) {
      const uint64_t x = __shfl_up_sync(0xFFFFFFFFu, incl, dd);
      if (lane >= (uint32_t)dd) incl += x;
    }
    uint8_t* h = d + base + incl - sz;
    if (sz) { *h++ = 0x0A; h += put_varint(h, len); }
    warp_copy_strings(h, f.data + s, len, sz != 0, UINT64_MAX);
    base += __shfl_sync(0xFFFFFFFFu, incl, 31);
  }
}
// The list payload of example i's bytes row (what ex_write_bytes writes), by the whole warp; flags request r in T.bad when the
// row breaks the offset rule.
__device__ __forceinline__ uint64_t ex_count_bytes(const ExTables& T, uint32_t r, const ExFeat& f, uint64_t i, uint64_t ne) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t b = i * f.row_stride;
  uint64_t lo, hi, carry, sum = 0;
  ex_row_bounds(f, b, &lo, &hi);
  carry = lo;
  bool bad = false;
  for (uint64_t j0 = 0; j0 < ne; j0 += 32) {
    uint64_t s;
    const uint64_t e = ex_str_ends(f, b, ne, j0, lo, hi, &carry, &s);
    const uint64_t j = j0 + lane;
    if (j < ne) {
      sum += string_value_len(e - s);
      bad |= f.offsets[b + j + 1] < f.offsets[b + j];
    }
  }
  if (lane == 0) {
    const int64_t o0 = f.offsets[b], on = f.offsets[b + ne], nx = f.offsets[b + f.row_elems];
    bad |= o0 < 0 || on > nx || nx > (int64_t)f.data_len;
  }
  if (__any_sync(0xFFFFFFFFu, bad) && lane == 0) T.bad[r] = 1;
  return warp_sum64(sum);
}

// Example i of request q, written by the calling warp at w (shared or global memory), behind the tag kTag: 0A
// (ExampleList.examples) or 42 (TensorProto.string_val).
template <int kMode, uint8_t kTag>
__device__ void ex_write_example(const ExTables& T, const ExReq& q, uint64_t i, uint8_t* w) {
  const uint32_t lane = threadIdx.x & 31;
  uint64_t F = 0, hl;
  for (uint32_t c = 0; c < q.n_feat; c += 32) {     // map entries, one feature per lane
    uint64_t e = 0;
    if (c + lane < q.n_feat) {
      const ExFeat& f = T.feats[q.first_feat + c + lane];
      e = ex_feat_entry_len<kMode>(f, ex_payload<kMode>(T, q, f, i), &hl);
    }
    F += warp_sum64(e);
  }
  const uint64_t X = 1 + varint_len(F) + F;
  uint64_t pos = 2 + varint_len(X) + varint_len(F);
  if (lane == 0) {
    w[0] = kTag;
    const uint32_t p = 1 + put_varint(w + 1, X);
    w[p] = 0x0A;
    put_varint(w + p + 1, F);
  }
  for (uint32_t c = 0; c < q.n_feat; c += 32) {
    const uint32_t k = c + lane;
    uint64_t e = 0, P = 0;
    hl = 0;
    if (k < q.n_feat) {
      const ExFeat f = T.feats[q.first_feat + k];
      P = ex_payload<kMode>(T, q, f, i);
      e = ex_feat_entry_len<kMode>(f, P, &hl);
    }
    uint64_t inc = e;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint64_t x = __shfl_up_sync(0xFFFFFFFFu, inc, d);
      if (lane >= (uint32_t)d) inc += x;
    }
    const uint64_t at = pos + inc - e;
    if (k < q.n_feat) {       // 0A vi(entry) 0A vi(klen) key 12 vi(Feature) {12|1A} vi(list) [0A vi(P)]   (bytes: 0A vi(P))
      const ExFeat& f = T.feats[q.first_feat + k];
      const bool str = kMode == kExColumns && f.op == EXO_BYTES;
      const uint64_t list = str ? P : P ? 1 + varint_len(P) + P : 0, feature = 1 + varint_len(list) + list;
      uint8_t* h = w + at;
      const uint64_t entry = 1 + varint_len(f.key_len) + f.key_len + 1 + varint_len(feature) + feature;
      *h++ = 0x0A; h += put_varint(h, entry);
      *h++ = 0x0A; h += put_varint(h, f.key_len);
      for (uint32_t b = 0; b < f.key_len; ++b) *h++ = T.blob[f.key_off + b];
      *h++ = 0x12; h += put_varint(h, feature);
      *h++ = str ? 0x0A : f.op < EXO_INT ? 0x12 : 0x1A; h += put_varint(h, list);
      if (P && !str) { *h++ = 0x0A; put_varint(h, P); }
    }
    const uint32_t nk = min(32u, q.n_feat - c);
    for (uint32_t s = 0; s < nk; ++s) {             // the rows, one after the other, by the whole warp
      const uint64_t Ps = __shfl_sync(0xFFFFFFFFu, P, s);
      const uint64_t ps = __shfl_sync(0xFFFFFFFFu, at + hl, s);
      if (!Ps) continue;
      const ExFeat f = T.feats[q.first_feat + c + s];
      const uint8_t* row = f.data + i * f.row_stride;
      const uint64_t ne = ex_elems<kMode>(f, i);
      uint8_t* d = w + ps;
      if (kMode == kExColumns && f.op == EXO_BYTES) {
        ex_write_bytes(f, i, ne, d);
      } else if (f.op < EXO_INT) {
        for (uint64_t j = lane; j < ne; j += 32) {
          const uint32_t b = ex_float_bits(f, row, j);
          d[4 * j] = (uint8_t)b; d[4 * j + 1] = (uint8_t)(b >> 8); d[4 * j + 2] = (uint8_t)(b >> 16); d[4 * j + 3] = (uint8_t)(b >> 24);
        }
      } else {
        uint64_t base = 0;
        for (uint64_t j0 = 0; j0 < ne; j0 += 32) {
          const uint64_t j = j0 + lane;
          uint64_t v = 0;
          uint32_t len = 0;
          if (j < ne) { v = ex_int(f, row + j * f.esz); len = vlen64(v); }
          uint32_t incl = len;
#pragma unroll
          for (int dd = 1; dd < 32; dd <<= 1) {
            const uint32_t x = __shfl_up_sync(0xFFFFFFFFu, incl, dd);
            if (lane >= (uint32_t)dd) incl += x;
          }
          if (len) put_varint(d + base + incl - len, v);
          base += __shfl_sync(0xFFFFFFFFu, incl, 31);
        }
      }
    }
    pos += __shfl_sync(0xFFFFFFFFu, inc, 31);
  }
}

template <int kMode>
__global__ void __launch_bounds__(kExTile) ex_count_kernel(const __grid_constant__ ExTables T) {
  __shared__ unsigned long long warp_sum[kExTile / 32];
  const ExSpan sp = T.tiles[blockIdx.x];
  const ExReq q = T.reqs[sp.req];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint64_t mine = 0;
  for (uint64_t i = sp.e0 + warp; i < sp.e1; i += kExTile / 32) {
    uint64_t F = 0, hl;
    for (uint32_t k = 0; k < q.n_feat; ++k) {
      const ExFeat f = T.feats[q.first_feat + k];
      const uint64_t ne = ex_elems<kMode>(f, i);
      if (kMode != kExDense && f.lengths && lane == 0) {      // compared, never multiplied: 2^62 must not wrap into range
        const int64_t l = f.lengths[i];
        if (l < 0 || (uint64_t)l > f.max_len) T.bad[sp.req] = 1;
      }
      uint64_t P = 4 * ne;
      if (kMode == kExColumns && f.op == EXO_BYTES) {
        P = ex_count_bytes(T, sp.req, f, i, ne);
        if (lane == 0) T.L[q.L0 + i * q.n_int + f.lcol] = P;
      } else if (f.op >= EXO_INT) {
        const uint8_t* row = f.data + i * f.row_stride;
        uint64_t s = 0;
        for (uint64_t j = lane; j < ne; j += 32) s += vlen64(ex_int(f, row + j * f.esz));
        P = warp_sum64(s);
        if (lane == 0) T.L[q.L0 + i * q.n_int + f.lcol] = P;
      }
      F += ex_feat_entry_len<kMode>(f, P, &hl);
    }
    const uint64_t S = ex_example_len(F);
    if (lane == 0) { T.S[q.ex0 + i] = S; mine += S; }
  }
  uint64_t total = 0;
  concat_scan(mine, total, warp_sum);
  if (threadIdx.x == 0) T.tile_sum[blockIdx.x] = total;
}

// ---- SequenceExamples (plan.h sq_*): a request's sequences take the place of its examples ----
// steps of sequence i of feature list f: a length clamped to [0, T] (the count kernel flags one that was not), or T
__device__ __forceinline__ uint64_t sq_steps(const ExFeat& f, uint64_t i) {
  if (!f.lengths) return f.max_len;
  const int64_t l = f.lengths[i];
  return l < 0 ? 0ull : min((uint64_t)l, f.max_len);
}
// ex_str_ends over strings j0 .. min(j0 + 32, ne) - 1 of a step whose last string is ne - 1: *carry moves on to the end of that
// last string, not to hi, so that the next step starts where this one ends
__device__ __forceinline__ uint64_t sq_str_ends(const ExFeat& f, uint64_t b, uint64_t ne, uint64_t j0, uint64_t lo, uint64_t hi,
                                                uint64_t* carry, uint64_t* start) {
  const uint64_t e = ex_str_ends(f, b, ne, j0, lo, hi, carry, start);
  *carry = __shfl_sync(0xFFFFFFFFu, e, (uint32_t)min(ne - j0, (uint64_t)32) - 1);
  return e;
}
// the list payload of step t of sequence i of list f (float: closed form; integer and bytes: the count kernel's)
__device__ __forceinline__ uint64_t sq_payload(const ExTables& T, const ExReq& q, const ExFeat& f, uint64_t i, uint64_t t) {
  return f.op < EXO_INT ? 4 * f.unit : T.L[q.L0 + i * q.n_int + f.lcol + t];
}
// the bytes of sequence i's steps of list f, by the whole warp
__device__ __forceinline__ uint64_t sq_list_len(const ExTables& T, const ExReq& q, const ExFeat& f, uint64_t i) {
  const uint64_t steps = sq_steps(f, i);
  if (f.op < EXO_INT) return steps * sq_step_len(4 * f.unit, false);
  uint64_t s = 0;
  for (uint64_t t = threadIdx.x & 31; t < steps; t += 32) s += sq_step_len(sq_payload(T, q, f, i, t), f.op == EXO_BYTES);
  return warp_sum64(s);
}

// One warp per sequence: the context as ex_count_kernel counts an example's features, and every step of every list, whose
// integer or bytes payload goes to its L column; a length or an offset out of range flags the request.
__global__ void __launch_bounds__(kExTile) ex_seq_count_kernel(const __grid_constant__ ExTables T) {
  __shared__ unsigned long long warp_sum[kExTile / 32];
  const ExSpan sp = T.tiles[blockIdx.x];
  const ExReq q = T.reqs[sp.req];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint64_t mine = 0;
  for (uint64_t i = sp.e0 + warp; i < sp.e1; i += kExTile / 32) {
    uint64_t C = 0, G = 0, hl;
    for (uint32_t k = 0; k < q.n_feat; ++k) {
      const ExFeat f = T.feats[q.first_feat + k];
      if (f.lengths && lane == 0) {      // compared, never multiplied: 2^62 must not wrap into range
        const int64_t l = f.lengths[i];
        if (l < 0 || (uint64_t)l > f.max_len) T.bad[sp.req] = 1;
      }
      uint64_t* L = T.L + q.L0 + i * q.n_int + f.lcol;
      if (k < q.n_ctx) {
        const uint64_t ne = ex_elems<kExColumns>(f, i);
        uint64_t P = 4 * ne;
        if (f.op == EXO_BYTES) {
          P = ex_count_bytes(T, sp.req, f, i, ne);
          if (lane == 0) *L = P;
        } else if (f.op >= EXO_INT) {
          const uint8_t* row = f.data + i * f.row_stride;
          uint64_t s = 0;
          for (uint64_t j = lane; j < ne; j += 32) s += vlen64(ex_int(f, row + j * f.esz));
          P = warp_sum64(s);
          if (lane == 0) *L = P;
        }
        C += ex_feat_entry_len<kExColumns>(f, P, &hl);
        continue;
      }
      const uint64_t steps = sq_steps(f, i), b = i * f.row_stride;
      uint64_t FL = 0;
      if (f.op < EXO_INT) {
        FL = steps * sq_step_len(4 * f.unit, false);
      } else if (f.op == EXO_BYTES) {      // ex_count_bytes over the sequence's row, one step after the other
        uint64_t lo, hi, carry;
        ex_row_bounds(f, b, &lo, &hi);
        carry = lo;
        bool bad = false;
        for (uint64_t t = 0; t < steps; ++t) {
          const uint64_t ne = (t + 1) * f.unit;
          uint64_t P = 0;
          for (uint64_t j0 = t * f.unit; j0 < ne; j0 += 32) {
            uint64_t s;
            const uint64_t e = sq_str_ends(f, b, ne, j0, lo, hi, &carry, &s), j = j0 + lane;
            if (j < ne) {
              P += string_value_len(e - s);
              bad |= f.offsets[b + j + 1] < f.offsets[b + j];
            }
          }
          P = warp_sum64(P);
          if (lane == 0) L[t] = P;
          FL += sq_step_len(P, true);
        }
        if (lane == 0) {
          const int64_t o0 = f.offsets[b], on = f.offsets[b + steps * f.unit], nx = f.offsets[b + f.row_elems];
          bad |= o0 < 0 || on > nx || nx > (int64_t)f.data_len;
        }
        if (__any_sync(0xFFFFFFFFu, bad) && lane == 0) T.bad[sp.req] = 1;
      } else {
        const uint8_t* row = f.data + b;
        for (uint64_t t = 0; t < steps; ++t) {
          uint64_t s = 0;
          for (uint64_t j = t * f.unit + lane; j < (t + 1) * f.unit; j += 32) s += vlen64(ex_int(f, row + j * f.esz));
          const uint64_t P = warp_sum64(s);
          if (lane == 0) L[t] = P;
          FL += sq_step_len(P, false);
        }
      }
      G += sq_list_entry_len(FL, f.key_len);
    }
    const uint64_t S = sq_sequence_len(C, G);
    if (lane == 0) { T.S[q.ex0 + i] = S; mine += S; }
  }
  uint64_t total = 0;
  concat_scan(mine, total, warp_sum);
  if (threadIdx.x == 0) T.tile_sum[blockIdx.x] = total;
}

// Sequence i of request q, written by the calling warp at w behind the tag 42.  The context is written by ex_write_example as an
// example of the context features, placed so that its `0A vi(C) entries` lands where the sequence has them: the example's own
// tag and length then lie inside the sequence's `42 vi(S)`, which lane 0 writes over them afterwards.
__device__ void ex_write_sequence(const ExTables& T, const ExReq& q, uint64_t i, uint8_t* w) {
  const uint32_t lane = threadIdx.x & 31;
  uint64_t C = 0, G = 0, hl;
  for (uint32_t c = 0; c < q.n_ctx; c += 32) {
    uint64_t e = 0;
    if (c + lane < q.n_ctx) {
      const ExFeat& f = T.feats[q.first_feat + c + lane];
      e = ex_feat_entry_len<kExColumns>(f, ex_payload<kExColumns>(T, q, f, i), &hl);
    }
    C += warp_sum64(e);
  }
  for (uint32_t k = q.n_ctx; k < q.n_feat; ++k) {
    const ExFeat& f = T.feats[q.first_feat + k];
    G += sq_list_entry_len(sq_list_len(T, q, f, i), f.key_len);
  }
  const uint64_t X = 1 + varint_len(C) + C + 1 + varint_len(G) + G, ctx_at = 1 + varint_len(X);
  ExReq qc = q;
  qc.n_feat = q.n_ctx;
  const uint64_t xc = 1 + varint_len(C) + C;             // the context example's X
  ex_write_example<kExColumns, 0x42>(T, qc, i, w + ctx_at - (1 + varint_len(xc)));
  uint64_t pos = ctx_at + xc;
  if (lane == 0) {
    w[0] = 0x42;
    put_varint(w + 1, X);
    w[pos] = 0x12;
    put_varint(w + pos + 1, G);
  }
  pos += 1 + varint_len(G);
  for (uint32_t k = q.n_ctx; k < q.n_feat; ++k) {
    const ExFeat f = T.feats[q.first_feat + k];
    const bool str = f.op == EXO_BYTES;
    const uint64_t FL = sq_list_len(T, q, f, i), steps = sq_steps(f, i);
    const uint64_t e = 1 + varint_len(f.key_len) + f.key_len + 1 + varint_len(FL) + FL;
    uint8_t* h = w + pos;        // 0A vi(e) 0A vi(klen) key 12 vi(FL)
    const uint32_t kat = 2 + varint_len(e) + varint_len(f.key_len);
    for (uint32_t b = lane; b < f.key_len; b += 32) h[kat + b] = T.blob[f.key_off + b];
    if (lane == 0) {
      h[0] = 0x0A; put_varint(h + 1, e);
      h[kat - 1 - varint_len(f.key_len)] = 0x0A; put_varint(h + kat - varint_len(f.key_len), f.key_len);
      h[kat + f.key_len] = 0x12; put_varint(h + kat + f.key_len + 1, FL);
    }
    pos += kat + f.key_len + 1 + varint_len(FL);
    const uint8_t* row = f.data + i * f.row_stride;
    if (f.op < EXO_INT) {        // every step the same size: headers one per lane, then the values one per lane
      const uint64_t P = 4 * f.unit, list = P ? 1 + varint_len(P) + P : 0, feat = 1 + varint_len(list) + list;
      const uint64_t sl = 1 + varint_len(feat) + feat, hd = sl - P;
      for (uint64_t t = lane; t < steps; t += 32) {     // 0A vi(feat) 12 vi(list) [0A vi(P)]
        uint8_t* s = w + pos + t * sl;
        *s++ = 0x0A; s += put_varint(s, feat);
        *s++ = 0x12; s += put_varint(s, list);
        if (P) { *s++ = 0x0A; put_varint(s, P); }
      }
      for (uint64_t j = lane; j < steps * f.unit; j += 32) {
        const uint64_t t = j / f.unit;
        const uint32_t v = ex_float_bits(f, row, j);
        uint8_t* d = w + pos + t * sl + hd + 4 * (j - t * f.unit);
        d[0] = (uint8_t)v; d[1] = (uint8_t)(v >> 8); d[2] = (uint8_t)(v >> 16); d[3] = (uint8_t)(v >> 24);
      }
      pos += steps * sl;
      continue;
    }
    uint64_t lo = 0, hi = 0, carry = 0;
    const uint64_t b = i * f.row_stride;
    if (str) { ex_row_bounds(f, b, &lo, &hi); carry = lo; }
    for (uint64_t t = 0; t < steps; ++t) {     // one step after the other, by the whole warp
      const uint64_t P = sq_payload(T, q, f, i, t), list = str ? P : P ? 1 + varint_len(P) + P : 0, feat = 1 + varint_len(list) + list;
      uint8_t* s = w + pos;
      const uint32_t hd = 1 + varint_len(feat) + (str ? 1 + varint_len(P) : P ? 2 + varint_len(list) + varint_len(P) : 1 + varint_len(list));
      if (lane == 0) {         // 0A vi(feat) {0A vi(P) | 1A vi(list) [0A vi(P)]}
        s[0] = 0x0A;
        uint32_t p = 1 + put_varint(s + 1, feat);
        s[p++] = str ? 0x0A : 0x1A;
        p += put_varint(s + p, str ? P : list);
        if (!str && P) { s[p++] = 0x0A; put_varint(s + p, P); }
      }
      uint8_t* d = s + hd;
      uint64_t base = 0;
      const uint64_t ne = (t + 1) * f.unit;
      for (uint64_t j0 = t * f.unit; j0 < ne; j0 += 32) {
        const uint64_t j = j0 + lane;
        uint64_t sz = 0, len = 0, st = 0, v = 0;
        if (str) {
          const uint64_t en = sq_str_ends(f, b, ne, j0, lo, hi, &carry, &st);
          len = j < ne ? en - st : 0;
          sz = j < ne ? string_value_len(len) : 0;
        } else if (j < ne) {
          v = ex_int(f, row + j * f.esz);
          sz = vlen64(v);
        }
        uint64_t incl = sz;
#pragma unroll
        for (int dd = 1; dd < 32; dd <<= 1) {
          const uint64_t x = __shfl_up_sync(0xFFFFFFFFu, incl, dd);
          if (lane >= (uint32_t)dd) incl += x;
        }
        uint8_t* o = d + base + incl - sz;
        if (str) {
          if (sz) { *o++ = 0x0A; o += put_varint(o, len); }
          warp_copy_strings(o, f.data + st, len, sz != 0, UINT64_MAX);
        } else if (sz) {
          put_varint(o, v);
        }
        base += __shfl_sync(0xFFFFFFFFu, incl, 31);
      }
      pos += 1 + varint_len(feat) + feat;
    }
  }
}

__global__ void __launch_bounds__(kExTile) ex_scan_kernel(const __grid_constant__ ExTables T) {
  __shared__ unsigned long long warp_sum[kExTile / 32];
  const uint32_t t = blockIdx.x;
  const ExSpan sp = T.tiles[t];
  const ExReq q = T.reqs[sp.req];
  uint64_t carry = 0;
  for (uint32_t k0 = q.first_tile; k0 < t; k0 += kExTile) {     // the tiles in front of this one (uniform trip count)
    const uint32_t k = k0 + threadIdx.x;
    concat_scan(k < t ? (uint64_t)T.tile_sum[k] : 0ull, carry, warp_sum);
  }
  const uint64_t i = sp.e0 + threadIdx.x;
  const uint64_t o = concat_scan(i < sp.e1 ? T.S[q.ex0 + i] : 0ull, carry, warp_sum);
  if (i < sp.e1) T.off[q.ex0 + i] = o;
}

// Does the scan place request q's examples?  Exactly when fixed_size == 0; without a ragged column that is when the request has an
// integer column, and the dense instantiation keeps that test (on sm_90a the other one costs its emit kernel 10 registers).
template <int kMode>
__device__ __forceinline__ bool ex_counted(const ExReq& q) {
  return kMode != kExDense ? q.fixed_size == 0 : q.n_int != 0;
}
// where example i of request q starts / ends, from the anchor
template <int kMode>
__device__ __forceinline__ uint64_t ex_start(const ExTables& T, const ExReq& q, uint64_t i) {
  return ex_counted<kMode>(q) ? T.off[q.ex0 + i] : i * q.fixed_size;
}
template <int kMode>
__device__ __forceinline__ uint64_t ex_end(const ExTables& T, const ExReq& q, uint64_t i) {
  return ex_counted<kMode>(q) ? T.off[q.ex0 + i] + T.S[q.ex0 + i] : (i + 1) * q.fixed_size;
}

// Store arena bytes [lo, hi) from the image img of the wire that starts at arena offset ws (16-byte aligned): the whole aligned
// vectors with 128-bit stores, the bytes of a partial vector at either end (which the neighbouring range shares) one by one.
__device__ __forceinline__ void ex_flush(uint8_t* arena, const uint8_t* img, uint64_t ws, uint64_t lo, uint64_t hi) {
  if (hi <= lo) return;
  const uint64_t a = min((uint64_t)((lo + 15) & ~15ull), hi), b = max((uint64_t)(hi & ~15ull), a);
  for (uint64_t x = lo + threadIdx.x; x < a; x += blockDim.x) arena[x] = img[x - ws];
  for (uint64_t x = a + 16ull * threadIdx.x; x < b; x += 16ull * blockDim.x)
    st_stream(arena + x, *reinterpret_cast<const uint4*>(img + (x - ws)));
  for (uint64_t x = b + threadIdx.x; x < hi; x += blockDim.x) arena[x] = img[x - ws];
}

// example i, or with kSeq sequence i, of request q at w
template <int kMode, uint8_t kTag, bool kSeq>
__device__ __forceinline__ void ex_write_record(const ExTables& T, const ExReq& q, uint64_t i, uint8_t* w) {
  if constexpr (kSeq) ex_write_sequence(T, q, i, w);
  else ex_write_example<kMode, kTag>(T, q, i, w);
}

// kShift (a PREDICT_ELWCS span, plan.h ExLists): the span's query (its pad) moves its examples by shift[query]; kEmpty (the
// device-planned spans, plan.h ExDevLists): an empty span writes nothing
template <int kMode, uint8_t kTag, bool kSeq = false, bool kShift = false, bool kEmpty = false>
__device__ __forceinline__ void ex_emit(const ExTables& T, const uint64_t* shift = nullptr) {
  __shared__ __align__(16) uint8_t img[kExStage + 16];
  __shared__ uint64_t next;
  constexpr uint32_t kWarps = kExEmitThreads / 32;
  const ExSpan sp = T.spans[blockIdx.x];
  if (kEmpty && sp.e1 <= sp.e0) return;
  const ExReq q = T.reqs[sp.req];
  const uint32_t warp = threadIdx.x >> 5;
  const uint64_t A = q.anchor + (kShift ? shift[sp.pad] : 0);
  // a bytes request whose offsets broke the rule can count more bytes than its slot holds (it gets B200TFS_E_SHAPE): a span
  // that would end past the slot writes nothing
  if ((kShift || kMode == kExColumns) && A + ex_end<kMode>(T, q, sp.e1 - 1) > q.slot_end) return;
  uint64_t lo = A + ex_start<kMode>(T, q, sp.e0);   // first byte not stored yet
  uint64_t ws = lo & ~15ull;                 // arena offset of img[0]
  uint64_t i = sp.e0;
  while (i < sp.e1) {
    if (threadIdx.x == 0) {                  // the longest run of examples from i whose bytes fit the image
      uint64_t g = i, h = sp.e1;
      while (g < h) {
        const uint64_t m = (g + h + 1) / 2;
        if (A + ex_end<kMode>(T, q, m - 1) - ws <= kExStage) g = m; else h = m - 1;
      }
      next = g;
    }
    __syncthreads();
    const uint64_t j = next;
    if (j > i) {
      for (uint64_t e = i + warp; e < j; e += kWarps) ex_write_record<kMode, kTag, kSeq>(T, q, e, img + (A + ex_start<kMode>(T, q, e) - ws));
      __syncthreads();
      const uint64_t be = A + ex_end<kMode>(T, q, j - 1), cut = be & ~15ull;
      if (cut > ws) {                        // store every whole vector; the partial one moves to the front of the image
        ex_flush(T.arena, img, ws, lo, cut);
        const uint8_t t = threadIdx.x < be - cut ? img[cut - ws + threadIdx.x] : 0;
        __syncthreads();
        if (threadIdx.x < be - cut) img[threadIdx.x] = t;
        ws = lo = cut;
      }
      i = j;
    } else {                                 // example i alone is larger than the image: one warp writes it in place
      ex_flush(T.arena, img, ws, lo, A + ex_start<kMode>(T, q, i));
      if (warp == 0) ex_write_record<kMode, kTag, kSeq>(T, q, i, T.arena + A + ex_start<kMode>(T, q, i));
      lo = A + ex_end<kMode>(T, q, i);
      ws = lo & ~15ull;
      ++i;
    }
    __syncthreads();
  }
  ex_flush(T.arena, img, ws, lo, A + ex_end<kMode>(T, q, sp.e1 - 1));
}

// The tag is a template argument, so the example_list kernels keep the registers they had before Predict requests existed.
template <int kMode>
__global__ void __launch_bounds__(kExEmitThreads) ex_emit_kernel(const __grid_constant__ ExTables T) {
  ex_emit<kMode, 0x0A>(T);
}
template <int kMode>
__global__ void __launch_bounds__(kExEmitThreads) ex_emit_predict_kernel(const __grid_constant__ ExTables T) {
  ex_emit<kMode, 0x42>(T);
}
// the spans of the PREDICT_ELWCS requests: their examples (kTag 0A, ExampleListWithContext.examples) and their contexts (12)
template <int kMode, uint8_t kTag>
__global__ void __launch_bounds__(kExEmitThreads) ex_emit_list_kernel(const __grid_constant__ ExTables T, const uint64_t* __restrict__ shift) {
  ex_emit<kMode, kTag, false, true>(T, shift);
}
// the example spans of the PREDICT_ELWCS requests with device list sizes, which ex_frame_lists_dev_kernel wrote (plan.h ExDevLists)
template <int kMode>
__global__ void __launch_bounds__(kExEmitThreads) ex_emit_list_dev_kernel(const __grid_constant__ ExTables T, const uint64_t* __restrict__ shift) {
  ex_emit<kMode, 0x0A, false, true, true>(T, shift);
}
// the spans of the SequenceExample requests, which are always counted (kExColumns places them through off and S)
__global__ void __launch_bounds__(kExEmitThreads) ex_emit_sequence_kernel(const __grid_constant__ ExTables T) {
  ex_emit<kExColumns, 0x42, true>(T);
}

constexpr uint32_t kExFrameWarps = 4;
// the bytes of request q's examples, by the calling warp
__device__ __forceinline__ uint64_t ex_examples_len(const ExTables& T, const ExReq& q) {
  const uint32_t lane = threadIdx.x & 31;
  uint64_t el = 0;
  if (!q.fixed_size) {
    for (uint32_t k = lane; k < q.n_tiles; k += 32) el += T.tile_sum[q.first_tile + k];
    el = warp_sum64(el);
  } else {
    el = q.n_ex * q.fixed_size;
  }
  return el;
}
// Request r's status, and when it is B200TFS_OK its prefix in front of the anchor, by the calling warp: el bytes of examples and
// `tail` bytes behind them (a context field), nested once more in a string_val with `nest` (Predict-ELWC); then the request's
// output_filter run (q.tail_len bytes of the blob) behind them.  bad: a length or an offset the request reads was out of range.
__device__ __forceinline__ int32_t ex_frame_request(const ExTables& T, const ExReq& q, uint32_t r, uint64_t el, uint64_t tail,
                                                    bool nest, bool bad) {
  const uint32_t lane = threadIdx.x & 31;
  // [00 be32(msg)] spec 12 vi(outer) mid inner_tag vi(inner) head [42 vi(body)] | body   (plan.h ExReq, ExCtxRef)
  const uint64_t body = el + tail, nested = nest ? 1 + varint_len(body) + body : body;
  const uint64_t inner = q.head_len + nested, outer = q.mid_len + 1 + varint_len(inner) + inner;
  const uint64_t msg = q.spec_len + 1 + varint_len(outer) + outer + q.tail_len;
  const uint64_t pre = (q.grpc ? 5 : 0) + msg - body - q.tail_len;
  int32_t st = B200TFS_OK;
  if (bad) st = B200TFS_E_SHAPE;
  else if (msg > 0x7FFFFFFFull) st = B200TFS_E_TOOBIG;
  else if (q.anchor + body + q.tail_len > q.slot_end) st = B200TFS_E_SIZE;
  if (lane == 0) {
    T.status[r] = st;
    T.rec_off[r] = st ? 0 : q.anchor - pre;
    T.rec_len[r] = st ? 0 : pre + body + q.tail_len;
  }
  if (st) return st;
  uint8_t* w = T.arena + q.anchor - pre;
  // the host-written bytes (spec, mid, head: one run in the blob) by the whole warp, the headers between them by lane 0
  const uint32_t at_spec = q.grpc ? 5 : 0, at_outer = at_spec + q.spec_len, at_mid = at_outer + 1 + varint_len(outer);
  const uint32_t at_inner = at_mid + q.mid_len, at_head = at_inner + 1 + varint_len(inner);
  for (uint32_t k = lane; k < q.spec_len + q.mid_len + q.head_len; k += 32) {
    const uint32_t d = k < q.spec_len ? at_spec + k : k < q.spec_len + q.mid_len ? at_mid + (k - q.spec_len) : at_head + (k - q.spec_len - q.mid_len);
    w[d] = T.blob[q.spec_off + k];
  }
  const uint32_t at_tail = q.spec_off + q.spec_len + q.mid_len + q.head_len;
  for (uint32_t k = lane; k < q.tail_len; k += 32) w[pre + body + k] = T.blob[at_tail + k];
  if (lane == 0) {
    if (q.grpc) { w[0] = 0; w[1] = (uint8_t)(msg >> 24); w[2] = (uint8_t)(msg >> 16); w[3] = (uint8_t)(msg >> 8); w[4] = (uint8_t)msg; }
    w[at_outer] = 0x12; put_varint(w + at_outer + 1, outer);
    w[at_inner] = (uint8_t)q.inner_tag; put_varint(w + at_inner + 1, inner);
    if (nest) { w[at_head + q.head_len] = 0x42; put_varint(w + at_head + q.head_len + 1, body); }
  }
  return st;
}

__global__ void __launch_bounds__(32 * kExFrameWarps) ex_frame_kernel(const __grid_constant__ ExTables T) {
  const uint32_t r = blockIdx.x * kExFrameWarps + (threadIdx.x >> 5);
  if (r >= T.n_req) return;
  const ExReq q = T.reqs[r];
  ex_frame_request(T, q, r, ex_examples_len(T, q), 0, false, T.bad && T.bad[r]);
}

// ex_frame_kernel for a call with contexts (plan.h ExCtxRef): a request with one also takes its context's size into its length,
// the context's bad flag into its status, and writes the context behind its examples, in place, with the request's warp
template <int kMode>
__device__ __forceinline__ void ex_frame_context(const ExTables& T, uint32_t r, const ExCtxRef c) {
  const uint32_t lane = threadIdx.x & 31;
  const ExReq q = T.reqs[r];
  const uint64_t el = ex_examples_len(T, q);
  if (c.req == kExNoContext) {
    ex_frame_request(T, q, r, el, 0, false, T.bad && T.bad[r]);
    return;
  }
  const ExReq x = T.reqs[c.req];
  const uint64_t cs = x.fixed_size ? x.fixed_size : T.S[x.ex0];    // the context field, its tag included
  if (ex_frame_request(T, q, r, el, cs, c.nest != 0, T.bad && (T.bad[r] || T.bad[c.req]))) return;
  uint8_t* w = T.arena + q.anchor + el;
  if (x.n_feat) ex_write_example<kMode, 0x12>(T, x, 0, w);
  else if (lane == 0) { w[0] = 0x12; w[1] = 0; }                 // context.SetInParent(): no features map at all
}
template <int kMode>
__global__ void __launch_bounds__(32 * kExFrameWarps) ex_frame_context_kernel(const __grid_constant__ ExTables T,
                                                                              const ExCtxRef* __restrict__ ctx) {
  const uint32_t r = blockIdx.x * kExFrameWarps + (threadIdx.x >> 5);
  if (r >= T.n_req) return;
  ex_frame_context<kMode>(T, r, ctx[r]);
}

// ex_frame_context_kernel for a call with a PREDICT_ELWCS request (plan.h ExLists), launched after the scan and before the emits:
// the warp of such a request walks its queries 32 at a time, one per lane.  Query q's examples take E_q bytes from their first
// contiguous offset, its context C_q (12 00 when empty); a warp scan of 1 + vi(E + C) + E + C gives where its header goes, which
// the lane writes, and the shifts the list emits move its examples and its context by.  No header leaves the slot, whatever the
// sizes: a request whose lengths or offsets broke the rules gets B200TFS_E_SHAPE, and its emits stop at the slot's end.
// kDev (D: plan.h ExDevLists): a request with device list sizes takes its queries from a warp scan of the sizes in the same loop,
// and writes its emit spans, a warp scan of ceil(size / per) placing each query's first one.
template <int kMode, bool kDev>
__device__ __forceinline__ void ex_frame_lists(const ExTables& T, const ExCtxRef* ctx, const ExLists& Ls, const ExDevLists* D) {
  const uint32_t r = blockIdx.x * kExFrameWarps + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= T.n_req) return;
  const ExCtxRef c = ctx[r];
  if (c.nest != kExListRef) {
    ex_frame_context<kMode>(T, r, c);
    return;
  }
  const ExList l = Ls.lists[c.req];
  const ExReq q = T.reqs[r], x = T.reqs[l.ctx];
  ExListSizes d{};
  if constexpr (kDev) d = D->lists[c.req];
  uint64_t base = 0;            // the bytes of the queries in front of this round
  uint64_t run = 0, used = 0;   // device sizes: the examples and the span slots of the queries in front of this round
  bool bad = false;             // and a negative size, or a sum past n_ex, in this lane's queries
  for (uint32_t k0 = 0; k0 < l.n_q; k0 += 32) {
    const uint32_t k = k0 + lane;
    uint64_t E = 0, C = 0, eo = 0, co = 0, h = 0;
    ExQuery e{0, 0};
    if (kDev && d.sizes) {      // the examples [e0, e1) clamped into [0, n_ex], and the spans over them
      const int64_t s = k < l.n_q ? d.sizes[k] : 0;
      const uint64_t z = s < 0 ? 0 : min((uint64_t)s, q.n_ex), zi = warp_incl_scan64(z);
      bad |= s < 0 || (uint64_t)s > q.n_ex || run + zi > q.n_ex;
      e.e0 = min(run + zi - z, q.n_ex); e.e1 = min(run + zi, q.n_ex);
      run = min(run + __shfl_sync(0xFFFFFFFFu, zi, 31), q.n_ex);
      const uint64_t ns = (e.e1 - e.e0 + d.per - 1) / d.per, ni = warp_incl_scan64(ns);
      ExSpan* sp = D->spans + d.s0 + used + (ni - ns);
      for (uint64_t j = 0; j < ns; ++j)
        sp[j] = ExSpan{r, l.q0 + k, e.e0 + j * d.per, min(e.e0 + (j + 1) * d.per, e.e1)};
      used += __shfl_sync(0xFFFFFFFFu, ni, 31);
    } else if (k < l.n_q) {
      e = Ls.queries[l.q0 + k];
    }
    if (k < l.n_q) {
      if (e.e1 > e.e0) { eo = ex_start<kMode>(T, q, e.e0); E = ex_end<kMode>(T, q, e.e1 - 1) - eo; }
      if (x.n_feat) { co = ex_start<kMode>(T, x, k); C = ex_end<kMode>(T, x, k) - co; }
      else C = 2;
      h = 1 + varint_len(E + C);
    }
    const uint64_t sz = h + E + C;
    uint64_t inc = sz;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint64_t y = __shfl_up_sync(0xFFFFFFFFu, inc, d);
      if (lane >= (uint32_t)d) inc += y;
    }
    const uint64_t P = base + inc - sz;     // the header, from the anchor
    if (k < l.n_q) {
      Ls.shift[l.q0 + k] = P + h - eo;
      Ls.cshift[l.q0 + k] = P + h + E - co;
      if (q.anchor + P + sz <= q.slot_end) {
        uint8_t* w = T.arena + q.anchor + P;
        w[0] = 0x42;
        put_varint(w + 1, E + C);
        if (!x.n_feat) { w[h + E] = 0x12; w[h + E + 1] = 0; }
      }
    }
    base += __shfl_sync(0xFFFFFFFFu, inc, 31);
  }
  if (kDev && d.sizes) {        // a bad request emits nothing; the slots behind the spans are empty
    bad = __any_sync(0xFFFFFFFFu, bad);
    if (bad) used = 0;
    for (uint64_t t = used + lane; t < d.n_s; t += 32) D->spans[d.s0 + t] = ExSpan{r, 0, 0, 0};
  }
  ex_frame_request(T, q, r, base, 0, false, (kDev && bad) || (T.bad && (T.bad[r] || T.bad[l.ctx])));
}
template <int kMode>
__global__ void __launch_bounds__(32 * kExFrameWarps) ex_frame_lists_kernel(const __grid_constant__ ExTables T,
                                                                            const ExCtxRef* __restrict__ ctx,
                                                                            const __grid_constant__ ExLists Ls) {
  ex_frame_lists<kMode, false>(T, ctx, Ls, nullptr);
}
// ex_frame_lists_kernel for a call with a PREDICT_ELWCS request whose list sizes are in device memory
template <int kMode>
__global__ void __launch_bounds__(32 * kExFrameWarps) ex_frame_lists_dev_kernel(const __grid_constant__ ExTables T,
                                                                                const ExCtxRef* __restrict__ ctx,
                                                                                const __grid_constant__ ExLists Ls,
                                                                                const __grid_constant__ ExDevLists D) {
  ex_frame_lists<kMode, true>(T, ctx, Ls, &D);
}

// n_seq_tiles / n_seq_spans: the count tiles and emit spans of the SequenceExample requests, behind T's n_tiles and n_spans
cudaError_t launch_example_requests(const ExTables& T, int mode, cudaStream_t stream, uint32_t* launched, const ExCtxRef* ctx,
                                    uint32_t n_seq_tiles, uint32_t n_seq_spans, const ExLists* lists, const ExDevLists* dev) {
  *launched = 0;
  if (T.n_tiles) {
    if (mode == kExColumns) ex_count_kernel<kExColumns><<<T.n_tiles, kExTile, 0, stream>>>(T);
    else if (mode == kExRagged) ex_count_kernel<kExRagged><<<T.n_tiles, kExTile, 0, stream>>>(T);
    else ex_count_kernel<kExDense><<<T.n_tiles, kExTile, 0, stream>>>(T);
    *launched += 1;
  }
  if (n_seq_tiles) {
    ExTables Q = T;
    Q.tiles += T.n_tiles;
    Q.tile_sum += T.n_tiles;
    ex_seq_count_kernel<<<n_seq_tiles, kExTile, 0, stream>>>(Q);
    *launched += 1;
  }
  if (T.n_tiles + n_seq_tiles) {      // the scan sees every tile: a request's tiles are contiguous, its first_tile global
    ex_scan_kernel<<<T.n_tiles + n_seq_tiles, kExTile, 0, stream>>>(T);
    *launched += 1;
  }
  const uint32_t frame_grid = (T.n_req + kExFrameWarps - 1) / kExFrameWarps;
  if (dev && T.n_req) {       // the shifts and the device-sized requests' spans (plan.h ExDevLists)
    if (mode == kExColumns) ex_frame_lists_dev_kernel<kExColumns><<<frame_grid, 32 * kExFrameWarps, 0, stream>>>(T, ctx, *lists, *dev);
    else if (mode == kExRagged) ex_frame_lists_dev_kernel<kExRagged><<<frame_grid, 32 * kExFrameWarps, 0, stream>>>(T, ctx, *lists, *dev);
    else ex_frame_lists_dev_kernel<kExDense><<<frame_grid, 32 * kExFrameWarps, 0, stream>>>(T, ctx, *lists, *dev);
    *launched += 1;
  } else if (lists && T.n_req) {     // the shifts, before every emit (plan.h ExLists)
    if (mode == kExColumns) ex_frame_lists_kernel<kExColumns><<<frame_grid, 32 * kExFrameWarps, 0, stream>>>(T, ctx, *lists);
    else if (mode == kExRagged) ex_frame_lists_kernel<kExRagged><<<frame_grid, 32 * kExFrameWarps, 0, stream>>>(T, ctx, *lists);
    else ex_frame_lists_kernel<kExDense><<<frame_grid, 32 * kExFrameWarps, 0, stream>>>(T, ctx, *lists);
    *launched += 1;
  }
  const uint32_t n_list = T.n_spans - T.n_predict_spans;
  if (n_list) {
    if (mode == kExColumns) ex_emit_kernel<kExColumns><<<n_list, kExEmitThreads, 0, stream>>>(T);
    else if (mode == kExRagged) ex_emit_kernel<kExRagged><<<n_list, kExEmitThreads, 0, stream>>>(T);
    else ex_emit_kernel<kExDense><<<n_list, kExEmitThreads, 0, stream>>>(T);
    *launched += 1;
  }
  if (T.n_predict_spans) {    // the spans of the Predict requests come last
    ExTables P = T;
    P.spans += n_list;
    if (mode == kExColumns) ex_emit_predict_kernel<kExColumns><<<T.n_predict_spans, kExEmitThreads, 0, stream>>>(P);
    else if (mode == kExRagged) ex_emit_predict_kernel<kExRagged><<<T.n_predict_spans, kExEmitThreads, 0, stream>>>(P);
    else ex_emit_predict_kernel<kExDense><<<T.n_predict_spans, kExEmitThreads, 0, stream>>>(P);
    *launched += 1;
  }
  if (n_seq_spans) {          // and those of the SequenceExample requests behind them
    ExTables Q = T;
    Q.spans += T.n_spans;
    ex_emit_sequence_kernel<<<n_seq_spans, kExEmitThreads, 0, stream>>>(Q);
    *launched += 1;
  }
  if (lists) {                // the spans of the PREDICT_ELWCS requests behind those: examples, then contexts
    ExTables Q = T;
    Q.spans += T.n_spans + n_seq_spans;
    if (lists->n_spans) {
      if (mode == kExColumns) ex_emit_list_kernel<kExColumns, 0x0A><<<lists->n_spans, kExEmitThreads, 0, stream>>>(Q, lists->shift);
      else if (mode == kExRagged) ex_emit_list_kernel<kExRagged, 0x0A><<<lists->n_spans, kExEmitThreads, 0, stream>>>(Q, lists->shift);
      else ex_emit_list_kernel<kExDense, 0x0A><<<lists->n_spans, kExEmitThreads, 0, stream>>>(Q, lists->shift);
      *launched += 1;
    }
    if (dev && dev->n_spans) {
      ExTables Qd = T;
      Qd.spans = dev->spans;
      if (mode == kExColumns) ex_emit_list_dev_kernel<kExColumns><<<dev->n_spans, kExEmitThreads, 0, stream>>>(Qd, lists->shift);
      else if (mode == kExRagged) ex_emit_list_dev_kernel<kExRagged><<<dev->n_spans, kExEmitThreads, 0, stream>>>(Qd, lists->shift);
      else ex_emit_list_dev_kernel<kExDense><<<dev->n_spans, kExEmitThreads, 0, stream>>>(Qd, lists->shift);
      *launched += 1;
    }
    Q.spans += lists->n_spans;
    if (lists->n_ctx_spans) {
      if (mode == kExColumns) ex_emit_list_kernel<kExColumns, 0x12><<<lists->n_ctx_spans, kExEmitThreads, 0, stream>>>(Q, lists->cshift);
      else if (mode == kExRagged) ex_emit_list_kernel<kExRagged, 0x12><<<lists->n_ctx_spans, kExEmitThreads, 0, stream>>>(Q, lists->cshift);
      else ex_emit_list_kernel<kExDense, 0x12><<<lists->n_ctx_spans, kExEmitThreads, 0, stream>>>(Q, lists->cshift);
      *launched += 1;
    }
    return cudaGetLastError();
  }
  if (T.n_req) {
    const uint32_t grid = frame_grid;
    if (!ctx) ex_frame_kernel<<<grid, 32 * kExFrameWarps, 0, stream>>>(T);
    else if (mode == kExColumns) ex_frame_context_kernel<kExColumns><<<grid, 32 * kExFrameWarps, 0, stream>>>(T, ctx);
    else if (mode == kExRagged) ex_frame_context_kernel<kExRagged><<<grid, 32 * kExFrameWarps, 0, stream>>>(T, ctx);
    else ex_frame_context_kernel<kExDense><<<grid, 32 * kExFrameWarps, 0, stream>>>(T, ctx);
    *launched += 1;
  }
  return cudaGetLastError();
}
