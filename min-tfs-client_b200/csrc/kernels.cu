// kernels.cu - sm_90a (H100) kernels of the TensorProto wire codec (pure HBM-bound byte packing: no
// tensor cores - see DESIGN.md "Roofline").
//
//   move_kernel{,_inline}  the pack/unpack engine: moves every payload between tensor memory and the
//                      wire arena (128-bit coalesced loads/stores, destination-aligned, a whole 32 KB
//                      tile in flight per CTA; a misaligned side is realigned in registers with funnel
//                      shifts, the neighbour block arriving by warp shuffle), applies the per-dtype
//                      fix-up (float32 sNaN quieting, bool normalisation, f16/bf16 <-> f32 casts)
//                      and writes the header fragments (tags, varint lengths, dims, keys).
//   decode_fused_kernel    a whole PredictResponse decode in one launch: framing-template check or
//                      tag walk (walker.h), destination layout, tile move, table to pinned host memory.
//   decode_fused_staged_kernel   the same for big batches (tiles of several 32 KB chunks): the tile's
//                      source bytes arrive by TMA 1-D bulk copies (cp.async.bulk global -> shared, two
//                      buffers, mbarrier completion) issued ahead of the template verdict.
//   decode_fused{,_staged}_cast_kernel   the same two with the narrowing tile move compiled in (b200tfs_set_decode_cast:
//                      float32 on the wire -> fp16 / bf16 in memory); mode 1 of the plain one is the VERIFY launch of the
//                      three-launch narrowing batch decode (two CTAs per record: verdict -> guard word, table).
//   move_guarded_kernel    the move engine over a host-built plan that stores only for records whose guard word is set.
//   parse_*_kernel     two-phase decode: one lane per PredictResponse / TensorProto walks the tags and
//                      tabulates dtype, dims and where the values lie.
//   frame_requests_kernel  deferred framing: one thread per request runs the framing writers (framing.h) over the device-side
//                      totals, writes every header byte, patches the destinations of the movers behind it.
//   ex_count / ex_scan / ex_emit / ex_frame_kernel   Classify / Regress requests: a batch of tf.Examples from columnar
//                      arrays (example_kernels.cuh).
//   xr_index / xr_scan / xr_emit / xr_compare / xr_publish_kernel   Classify / Regress responses: a batch of responses into
//                      one value / score array (example_resp_kernels.cuh, walk in example_walk.h).
//   mi_index_kernel    MultiInference responses: assigns each result's entries to its task, whose view the xr kernels then
//                      decode (multi_resp_kernels.cuh, walk in multi_walk.h).
//   venc_* / vdec_*    packed-varint encode and decode (int_val / int64_val / uint32_val / uint64_val /
//                      half_val / bool_val): varint_kernels.cuh.  vdec_plan_kernel + vdec_{count,emit}_dev_kernel decode the
//                      varint outputs of a single-launch decode from tables built on the device (b200tfs_set_decode_varints).
//
// What the reference does at these points: tensors.py:22 (per-element .item() loop feeding
// RepeatedScalarContainer.extend), prediction_service_pb2_grpc.py:52-53 (SerializeToString /
// FromString in the protobuf runtime), tensors.py:46 (per-element list -> np.array).
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <utility>

#include "framing.h"
#include "kernels.h"
#include "plan.h"
#include "strcol.h"
#include "string_walk.h"
#include "tpl.h"
#include "unpad.h"
#include "example_walk.h"
#include "multi_walk.h"
#include "walker.h"
#include "wire.h"

namespace b200tfs {

// ------------------------------------------------------------------------------------------------
// 128-bit global accessors
// ------------------------------------------------------------------------------------------------
// streaming load: read once, do not keep in L1
__device__ __forceinline__ uint4 ld_stream(const uint8_t* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
// load that may allocate in L1: the shifted path reads every 16-byte block twice (as `lo` of one
// vector and `hi` of its neighbour), the second read should hit L1
__device__ __forceinline__ uint4 ld_reuse(const uint8_t* p) {
  uint4 r;
  asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ void st_stream(uint8_t* p, const uint4& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};"
               :: "l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// Programmatic dependent launch: let the NEXT kernel of the stream start launching right away, and
// hold our own memory accesses until every earlier kernel has completed and flushed.  Both are no-ops
// unless the launch carries cudaLaunchAttributeProgrammaticStreamSerialization (launch_pdl below), in
// which case the launch ramp of kernel N+1 overlaps the tail of kernel N instead of following it.
// Ordering and visibility are unchanged.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait_prior_grids() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

__device__ __forceinline__ uint32_t bool_norm_word(uint32_t w) {
  // per byte: b != 0 -> 1
  uint32_t t = ((w & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | w;
  return (t >> 7) & 0x01010101u;
}

template <uint32_t OP>
__device__ __forceinline__ uint4 fix_vec(uint4 v) {
  if (OP == OP_QUIET_SRC || OP == OP_QUIET_DST) {
    v.x = quiet_f32(v.x); v.y = quiet_f32(v.y); v.z = quiet_f32(v.z); v.w = quiet_f32(v.w);
  } else if (OP == OP_BOOL) {
    v.x = bool_norm_word(v.x); v.y = bool_norm_word(v.y); v.z = bool_norm_word(v.z); v.w = bool_norm_word(v.w);
  }
  return v;
}

// bytes [k, k+16) of the 32-byte little-endian concatenation lo:hi, k = 4*Q + s/8, 0 < k < 16
template <int Q>
__device__ __forceinline__ uint4 shift_pair(const uint4& lo, const uint4& hi, uint32_t s) {
  const uint32_t w[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
  uint4 o;
  o.x = __funnelshift_r(w[Q + 0], w[Q + 1], s);
  o.y = __funnelshift_r(w[Q + 1], w[Q + 2], s);
  o.z = __funnelshift_r(w[Q + 2], w[Q + 3], s);
  o.w = __funnelshift_r(w[Q + 3], w[Q + 4], s);
  return o;
}

// ------------------------------------------------------------------------------------------------
// element-exact byte generator: byte i of the output stream of `op` applied to src.  Used for the
// ragged head / tail of every payload, for small items, and as the fallback when a payload's
// alignment does not qualify for a vector path.  Alignment-agnostic by construction.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t ld_u32_bytes(const uint8_t* p) {
  return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}
__device__ __forceinline__ uint32_t f16_bits_to_f32_bits(uint32_t h) {
  return __float_as_uint(__half2float(__ushort_as_half((unsigned short)h)));
}
// widening casts follow IEEE-754 convertFormat: NaNs come out quiet with sign and payload kept
// (what numpy's astype(float32) followed by the reference's float32 round trip produces)
__device__ __forceinline__ uint32_t widen_f16(uint32_t h) {
  if ((h & 0x7C00u) == 0x7C00u && (h & 0x3FFu)) return ((h & 0x8000u) << 16) | 0x7FC00000u | ((h & 0x3FFu) << 13);
  return f16_bits_to_f32_bits(h);
}
__device__ __forceinline__ uint32_t widen_bf16(uint32_t h) { return quiet_f32(h << 16); }
// narrowing casts give what numpy's astype(float16) / ml_dtypes' astype(bfloat16) give for the float32 the reference
// decodes, whose NaNs are quiet: float16 keeps the sign and the top ten payload bits of the quieted NaN, bfloat16 writes
// the quiet NaN with the sign kept.  cvt.rn.{f16,bf16}.f32 alone would turn every NaN into 0x7FFF.
__device__ __forceinline__ uint32_t f32_bits_to_f16_bits(uint32_t w) {
  if ((w & 0x7FFFFFFFu) > 0x7F800000u) return ((w >> 16) & 0x8000u) | 0x7E00u | ((w >> 13) & 0x3FFu);
  return (uint32_t)__half_as_ushort(__float2half_rn(__uint_as_float(w)));
}
__device__ __forceinline__ uint32_t f32_bits_to_bf16_bits(uint32_t w) {
  if ((w & 0x7FFFFFFFu) > 0x7F800000u) return ((w >> 16) & 0x8000u) | 0x7FC0u;
  return (uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(__uint_as_float(w)));
}

// the logical source byte stream of an item: contiguous memory, or (gstride != 0) a row of pieces of `glen` value bytes
// every `gstride` bytes - a run of unpacked elements on the wire (b200tfs_run)
struct SrcView {
  const uint8_t* p;
  uint32_t glen, gstride;
  __device__ __forceinline__ uint8_t operator[](uint64_t j) const {
    if (gstride == 0) return p[j];
    const uint64_t q = j / glen;
    return p[q * gstride + (j - q * glen)];
  }
  __device__ __forceinline__ uint32_t u32(uint64_t j) const {
    return (uint32_t)(*this)[j] | ((uint32_t)(*this)[j + 1] << 8) | ((uint32_t)(*this)[j + 2] << 16) | ((uint32_t)(*this)[j + 3] << 24);
  }
};

__device__ __forceinline__ uint8_t gen_byte(uint32_t op, const SrcView& src, uint64_t i) {
  switch (op) {
    case OP_COPY: return src[i];
    case OP_BOOL: return src[i] != 0;
    case OP_QUIET_SRC:
    case OP_QUIET_DST: {
      uint32_t w = quiet_f32(src.u32(i & ~3ull));
      return (uint8_t)(w >> (8 * (i & 3)));
    }
    case OP_H2F: {
      uint64_t e = i >> 2;
      uint32_t h = (uint32_t)src[2 * e] | ((uint32_t)src[2 * e + 1] << 8);
      return (uint8_t)(widen_f16(h) >> (8 * (i & 3)));
    }
    case OP_B2F: {
      uint64_t e = i >> 2;
      uint32_t h = (uint32_t)src[2 * e] | ((uint32_t)src[2 * e + 1] << 8);
      return (uint8_t)(widen_bf16(h) >> (8 * (i & 3)));
    }
    case OP_F2H: {
      uint64_t e = i >> 1;
      return (uint8_t)(f32_bits_to_f16_bits(src.u32(4 * e)) >> (8 * (i & 1)));
    }
    case OP_F2B: {
      uint64_t e = i >> 1;
      return (uint8_t)(f32_bits_to_bf16_bits(src.u32(4 * e)) >> (8 * (i & 1)));
    }
  }
  return 0;
}
__device__ __forceinline__ uint8_t gen_byte(uint32_t op, const uint8_t* src, uint64_t i) { return gen_byte(op, SrcView{src, 0u, 0u}, i); }

// source bytes consumed per output byte, as a ratio num/den
__device__ __forceinline__ uint64_t src_bytes_for(uint32_t op, uint64_t n_out) {
  if (op == OP_H2F || op == OP_B2F) return n_out >> 1;
  if (op == OP_F2H || op == OP_F2B) return n_out << 1;
  return n_out;
}

// ------------------------------------------------------------------------------------------------
// vector bodies.  `src` / `dst` point at the first byte of the TILE's body; n = destination vectors
// in the tile.  Every thread issues all loads of a batch (kBatchAligned / kBatchShift vectors) before its first store:
// a 4 MiB tensor is smaller than the HBM bandwidth-delay product, so the whole tile must be in
// flight at once - one DRAM round trip per batch, not per vector.
// ------------------------------------------------------------------------------------------------

constexpr uint32_t kBatchAligned = 8;  // aligned path: 8 x 16 B per thread = a 32 KB tile in one round trip

// `mid` runs once per thread after the FIRST round's loads are in flight and before any store; it
// returns false to abandon the tile (the fused decode's template verdict, which needs a DRAM round
// trip of its own, hides behind the tile's loads this way).  Plain callers pass AlwaysGo.
struct AlwaysGo { __device__ __forceinline__ bool operator()() const { return true; } };

template <uint32_t OP, class Mid>
__device__ __forceinline__ bool body_aligned(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, uint32_t n, Mid& mid) {
  for (uint32_t base = 0; base < n; base += kBatchAligned * kMoveThreads) {   // uniform trip count across the CTA
    const uint32_t v = base + threadIdx.x;
    uint4 a[kBatchAligned];
#pragma unroll
    for (uint32_t i = 0; i < kBatchAligned; ++i)
      if (v + i * kMoveThreads < n) a[i] = ld_stream(src + 16ull * (v + i * kMoveThreads));
    if (base == 0 && !mid()) return false;
#pragma unroll
    for (uint32_t i = 0; i < kBatchAligned; ++i)
      if (v + i * kMoveThreads < n) st_stream(dst + 16ull * (v + i * kMoveThreads), fix_vec<OP>(a[i]));
  }
  return true;
}

// S = source body rounded down to 16 bytes; output vector v = bytes [k, k+16) of blocks v, v+1.
// Each source block is loaded ONCE: lane L takes block v+1 from lane L+1 by shuffle (lane 31, and
// the last lane of a ragged tile, load it themselves: +1/32 traffic).  ncu showed why: two loads
// of the same block in flight together are not merged - both go to DRAM.
__device__ __forceinline__ uint4 shfl_down1(const uint4& v) {
  uint4 r;
  r.x = __shfl_down_sync(0xFFFFFFFFu, v.x, 1); r.y = __shfl_down_sync(0xFFFFFFFFu, v.y, 1);
  r.z = __shfl_down_sync(0xFFFFFFFFu, v.z, 1); r.w = __shfl_down_sync(0xFFFFFFFFu, v.w, 1);
  return r;
}

__device__ __forceinline__ uint4 shfl_lane0(const uint4& v) {
  uint4 r;
  r.x = __shfl_sync(0xFFFFFFFFu, v.x, 0); r.y = __shfl_sync(0xFFFFFFFFu, v.y, 0);
  r.z = __shfl_sync(0xFFFFFFFFu, v.z, 0); r.w = __shfl_sync(0xFFFFFFFFu, v.w, 0);
  return r;
}

// Each WARP owns a contiguous run of kBatchShift*32 destination vectors: element i of lane L is vector
// run + 32*i + L.  Block v+1 then comes from lane L+1 (shuffle), for lane 31 from lane 0's NEXT
// element, and only the block just past the run is loaded extra (by lane 0).  All kBatchShift loads
// of a thread are in flight together: a 32 KB tile is one DRAM round trip, like the aligned path.
constexpr uint32_t kBatchShift = 8;

template <uint32_t OP, int Q, class Mid>
__device__ __forceinline__ bool body_shifted_q(const uint8_t* __restrict__ S, uint8_t* __restrict__ dst, uint32_t n, uint32_t s, Mid& mid) {
  constexpr bool PRE = (OP == OP_QUIET_SRC);  // elements line up with the source blocks
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  constexpr uint32_t kRun = kBatchShift * 32;                    // vectors per warp per round
  constexpr uint32_t kRound = kRun * (kMoveThreads / 32);        // vectors per CTA per round
  for (uint32_t base = 0; base < n; base += kRound) {            // uniform trip count across the CTA
    const uint32_t run = base + warp * kRun;
    const uint32_t run_end = min(run + kRun, n);                 // first vector past this warp's run (block index of `extra`)
    uint4 lo[kBatchShift], extra = make_uint4(0, 0, 0, 0);
#pragma unroll
    for (uint32_t i = 0; i < kBatchShift; ++i) {
      const uint32_t u = run + 32 * i + lane;
      lo[i] = make_uint4(0, 0, 0, 0);
      if (u < n) lo[i] = ld_stream(S + 16ull * u);
    }
    if (lane == 0 && run < n) extra = ld_stream(S + 16ull * run_end);
    if (base == 0 && !mid()) return false;
    extra = shfl_lane0(extra);
#pragma unroll
    for (uint32_t i = 0; i < kBatchShift; ++i) {
      const uint32_t u = run + 32 * i + lane;
      uint4 b = shfl_down1(lo[i]);                               // lanes 0..30: neighbour's block
      if (i + 1 < kBatchShift) {
        const uint4 nxt = shfl_lane0(lo[i + 1]);                 // lane 31: first block of the next element
        if (lane == 31) b = nxt;
      }
      if (u + 1 == run_end) b = extra;                           // last vector of the run (or of a ragged tile)
      if (u < n) {
        uint4 a = lo[i];
        if (PRE) { a = fix_vec<OP>(a); b = fix_vec<OP>(b); }
        uint4 o = shift_pair<Q>(a, b, s);
        if (!PRE) o = fix_vec<OP>(o);
        st_stream(dst + 16ull * u, o);
      }
    }
  }
  return true;
}

template <uint32_t OP, class Mid>
__device__ __forceinline__ bool body_same_width(const uint8_t* src, uint8_t* dst, uint32_t n, Mid& mid) {
  const uint32_t k = (uint32_t)((uintptr_t)src & 15);
  if (k == 0) return body_aligned<OP>(src, dst, n, mid);
  const uint8_t* S = src - k;
  const uint32_t s = (k & 3) * 8;
  switch (k >> 2) {  // uniform across the CTA
    case 0: return body_shifted_q<OP, 0>(S, dst, n, s, mid);
    case 1: return body_shifted_q<OP, 1>(S, dst, n, s, mid);
    case 2: return body_shifted_q<OP, 2>(S, dst, n, s, mid);
    default: return body_shifted_q<OP, 3>(S, dst, n, s, mid);
  }
}

// f16 / bf16 -> f32 (encode-side cast).  Both sides 16-byte aligned; unit u = 16 source bytes -> 32 out.  Eight loads per thread
// are in flight before the first store, like the same-width bodies (two were too few to cover DRAM latency).
template <bool BF>
__device__ __forceinline__ void body_widen(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, uint32_t units) {
  constexpr uint32_t kU = 8;
  for (uint32_t base = 0; base < units; base += kU * kMoveThreads) {      // uniform trip count across the CTA
    uint4 h[kU];
#pragma unroll
    for (uint32_t i = 0; i < kU; ++i) {
      const uint32_t u = base + i * kMoveThreads + threadIdx.x;
      h[i] = make_uint4(0, 0, 0, 0);
      if (u < units) h[i] = ld_stream(src + 16ull * u);
    }
#pragma unroll
    for (uint32_t i = 0; i < kU; ++i) {
      const uint32_t u = base + i * kMoveThreads + threadIdx.x;
      if (u < units) {
        const uint4 x = h[i];
        uint4 lo, hi;
        if (BF) {
          lo.x = widen_bf16(x.x & 0xFFFF); lo.y = widen_bf16(x.x >> 16); lo.z = widen_bf16(x.y & 0xFFFF); lo.w = widen_bf16(x.y >> 16);
          hi.x = widen_bf16(x.z & 0xFFFF); hi.y = widen_bf16(x.z >> 16); hi.z = widen_bf16(x.w & 0xFFFF); hi.w = widen_bf16(x.w >> 16);
        } else {
          lo.x = widen_f16(x.x & 0xFFFF); lo.y = widen_f16(x.x >> 16); lo.z = widen_f16(x.y & 0xFFFF); lo.w = widen_f16(x.y >> 16);
          hi.x = widen_f16(x.z & 0xFFFF); hi.y = widen_f16(x.z >> 16); hi.z = widen_f16(x.w & 0xFFFF); hi.w = widen_f16(x.w >> 16);
        }
        st_stream(dst + 32ull * u, lo);
        st_stream(dst + 32ull * u + 16, hi);
      }
    }
  }
}

// f32 -> f16 / bf16 (decode-side cast).  dst 16-byte aligned; source any alignment.
template <bool BF>
__device__ __forceinline__ uint32_t narrow2(uint32_t a, uint32_t b) {
  return BF ? (f32_bits_to_bf16_bits(a) | (f32_bits_to_bf16_bits(b) << 16))
            : (f32_bits_to_f16_bits(a) | (f32_bits_to_f16_bits(b) << 16));
}
// Output vector u (8 halfs) <- source blocks 2u, 2u+1 (+ 2u+2 when the source is shifted).  Every warp owns a contiguous run of
// 32 * kU output vectors per round, so that block 2u+2 is the neighbour lane's block 2(u+1) - by shuffle - and only the run's
// last vector needs a load of its own; all 2 * kU (+1) loads of a thread are issued before its first store (with two vectors per
// thread too few bytes are in flight per SM to cover DRAM latency).
// `mid` runs once, between the first round's loads and its stores (the fused decode's framing verdict: nothing may be stored
// before it, but the tile's bytes can already be on their way).
template <bool BF, int Q, class Mid>
__device__ __forceinline__ bool body_narrow_q(const uint8_t* __restrict__ S, uint8_t* __restrict__ dst, uint32_t n, uint32_t s, bool aligned, Mid& mid) {
  constexpr uint32_t kU = 4, kRun = 32 * kU, kRound = kRun * (kMoveThreads / 32);
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (uint32_t base = 0; base < n; base += kRound) {                      // uniform trip count across the CTA
    const uint32_t run = base + warp * kRun;
    const uint32_t run_end = min(run + kRun, n);
    uint4 a[kU], b[kU], extra = make_uint4(0, 0, 0, 0);
#pragma unroll
    for (uint32_t i = 0; i < kU; ++i) {
      const uint32_t u = run + 32 * i + lane;
      a[i] = b[i] = make_uint4(0, 0, 0, 0);
      if (u < n) { const uint8_t* p = S + 32ull * u; a[i] = ld_stream(p); b[i] = ld_stream(p + 16); }
    }
    if (!aligned && lane == 0 && run < n) extra = ld_stream(S + 32ull * run_end);     // the block behind the run's last vector
    if (base == 0 && !mid()) return false;
    extra = shfl_lane0(extra);
#pragma unroll
    for (uint32_t i = 0; i < kU; ++i) {
      const uint32_t u = run + 32 * i + lane;
      uint4 c = shfl_down1(a[i]);                                  // lanes 0..30: the neighbour's first block
      if (i + 1 < kU) {
        const uint4 nxt = shfl_lane0(a[i + 1]);                    // lane 31: first block of the next row of this run
        if (lane == 31) c = nxt;
      }
      if (u + 1 == run_end) c = extra;
      if (u < n) {
        uint4 f0 = a[i], f1 = b[i];
        if (!aligned) { f0 = shift_pair<Q>(a[i], b[i], s); f1 = shift_pair<Q>(b[i], c, s); }
        uint4 o;
        o.x = narrow2<BF>(f0.x, f0.y); o.y = narrow2<BF>(f0.z, f0.w);
        o.z = narrow2<BF>(f1.x, f1.y); o.w = narrow2<BF>(f1.z, f1.w);
        st_stream(dst + 16ull * u, o);
      }
    }
  }
  return true;
}

template <bool BF, class Mid>
__device__ __forceinline__ bool body_narrow(const uint8_t* src, uint8_t* dst, uint32_t n, Mid& mid) {
  const uint32_t k = (uint32_t)((uintptr_t)src & 15);
  const uint8_t* S = src - k;
  const uint32_t s = (k & 3) * 8;
  switch (k >> 2) {
    case 0: return body_narrow_q<BF, 0>(S, dst, n, s, k == 0, mid);
    case 1: return body_narrow_q<BF, 1>(S, dst, n, s, false, mid);
    case 2: return body_narrow_q<BF, 2>(S, dst, n, s, false, mid);
    default: return body_narrow_q<BF, 3>(S, dst, n, s, false, mid);
  }
}

// ------------------------------------------------------------------------------------------------
// one tile of one large payload.  Geometry in destination space: [head bytes][nvec vectors][tail];
// tile t owns vectors [t*vpt, (t+1)*vpt); tile 0 also writes the head, the last tile the tail.
// ------------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ uint32_t tiles_for(uint64_t n_out, uint32_t vpt) {
  const uint64_t vecs = (n_out + 15) >> 4;
  const uint64_t t = (vecs + vpt - 1) / vpt;
  return t ? (uint32_t)t : 1u;
}

// a gathered source (a run of unpacked elements): element-exact byte path, split by tile
__device__ __forceinline__ void move_tile_gather(const SrcView& src, uint8_t* __restrict__ dst, uint64_t n_out, uint32_t op, uint32_t n_tiles,
                                                 uint32_t tile, uint32_t vpt) {
  const uint64_t b0 = (uint64_t)tile * vpt * 16;
  uint64_t b1 = b0 + (uint64_t)vpt * 16;
  if (b1 > n_out || tile + 1 == n_tiles) b1 = n_out;
  for (uint64_t i = b0 + threadIdx.x; i < b1; i += blockDim.x) dst[i] = gen_byte(op, src, i);
}

// DEC: the caller only ever passes OP_COPY / OP_QUIET_DST (the single-launch decode moves float_val / double_val / complex
// values as they are): the other bodies are not instantiated there (with every body inlined three times the fused decode kernel
// was 728 KB of SASS).  The narrowing decode (CAST instantiations, move_guarded_kernel) goes through DEC = false.
template <bool DEC, class Mid>
__device__ __forceinline__ bool move_tile(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, uint64_t n_out, uint32_t op,
                                          uint32_t n_tiles, uint32_t tile, uint32_t vpt, Mid& mid) {
  const bool last = (tile + 1 == n_tiles);
  const uint64_t n_src = DEC ? n_out : src_bytes_for(op, n_out);
  uint64_t head = (16 - ((uintptr_t)dst & 15)) & 15;
  if (head > n_out) head = n_out;
  bool fast = true;
  uint64_t nvec;                 // destination vectors a vector path may handle
  const uint8_t* src_body = src + head;
  if (DEC || op <= OP_QUIET_DST || op == OP_BOOL) {      // same width
    if (!DEC && op == OP_QUIET_SRC) fast = (((uintptr_t)src & 3) == 0);
    if (op == OP_QUIET_DST) fast = ((head & 3) == 0);
    nvec = (n_out - head) >> 4;
    const uint32_t k = (uint32_t)((uintptr_t)src_body & 15);
    if (k) {  // the shifted path also reads block v+1: keep that inside the source
      const uint64_t blocks = (uint64_t)((src + n_src) - (src_body - k)) >> 4;
      const uint64_t lim = blocks ? blocks - 1 : 0;
      if (nvec > lim) nvec = lim;
    }
  } else if (op == OP_H2F || op == OP_B2F) {
    src_body = src;
    fast = (head == 0) && (((uintptr_t)src & 15) == 0);
    nvec = (n_out >> 5) << 1;    // whole 32-byte units, counted in 16-byte vectors
  } else {                       // OP_F2H / OP_F2B
    src_body = src + 2 * head;
    fast = ((head & 1) == 0);
    nvec = (n_out - head) >> 4;
    const uint32_t k = (uint32_t)((uintptr_t)src_body & 15);
    const uint64_t span = (uint64_t)((src + n_src) - (src_body - k));
    const uint64_t lim = k ? (span >= 16 ? (span - 16) >> 5 : 0) : (span >> 5);
    if (nvec > lim) nvec = lim;
  }
  if (!fast) {  // whole payload through the byte generator, split by tile
    if (!mid()) return false;
    const uint64_t b0 = (uint64_t)tile * vpt * 16;
    uint64_t b1 = b0 + (uint64_t)vpt * 16;
    if (b1 > n_out || last) b1 = n_out;
    for (uint64_t i = b0 + threadIdx.x; i < b1; i += blockDim.x) dst[i] = gen_byte(op, src, i);
    return true;
  }
  const uint64_t v0 = (uint64_t)tile * vpt;
  bool go;
  if (v0 < nvec) {
    const uint32_t n = (uint32_t)min((uint64_t)vpt, nvec - v0);
    uint8_t* d = dst + head + 16 * v0;
    if (DEC) {
      if (op == OP_COPY) go = body_same_width<OP_COPY>(src_body + 16 * v0, d, n, mid);
      else go = body_same_width<OP_QUIET_DST>(src_body + 16 * v0, d, n, mid);
    } else {
      switch (op) {
        case OP_COPY: go = body_same_width<OP_COPY>(src_body + 16 * v0, d, n, mid); break;
        case OP_BOOL: go = body_same_width<OP_BOOL>(src_body + 16 * v0, d, n, mid); break;
        case OP_QUIET_SRC: go = body_same_width<OP_QUIET_SRC>(src_body + 16 * v0, d, n, mid); break;
        case OP_QUIET_DST: go = body_same_width<OP_QUIET_DST>(src_body + 16 * v0, d, n, mid); break;
        case OP_H2F: go = mid(); if (go) body_widen<false>(src_body + 8 * v0, d, n >> 1); break;
        case OP_B2F: go = mid(); if (go) body_widen<true>(src_body + 8 * v0, d, n >> 1); break;
        case OP_F2H: go = body_narrow<false>(src_body + 32 * v0, d, n, mid); break;
        default: go = body_narrow<true>(src_body + 32 * v0, d, n, mid); break;
      }
    }
  } else go = mid();
  if (!go) return false;
  // ragged edges, element-exact
  if (tile == 0) for (uint64_t i = threadIdx.x; i < head; i += blockDim.x) dst[i] = gen_byte(op, src, i);
  if (last) for (uint64_t i = head + (nvec << 4) + threadIdx.x; i < n_out; i += blockDim.x) dst[i] = gen_byte(op, src, i);
  return true;
}

// ------------------------------------------------------------------------------------------------
// one out-of-line copy of the decode-side tile move for the paths where speed is not the point (a walked record, a staged
// tile whose geometry does not qualify): called, not inlined, so that the hot paths stay compact
__device__ __noinline__ void move_tile_cold(const uint8_t* src, uint8_t* dst, uint64_t n_out, uint32_t op, uint32_t n_tiles, uint32_t tile,
                                            uint32_t vpt) {
  AlwaysGo go;
  move_tile<true>(src, dst, n_out, op, n_tiles, tile, vpt, go);
}

// the narrowing ops (float32 on the wire -> fp16 / bf16 in memory: b200tfs_set_decode_cast) through the general tile move, out of line
__device__ __noinline__ void move_tile_narrow(const uint8_t* src, uint8_t* dst, uint64_t n_out, uint32_t op, uint32_t n_tiles, uint32_t tile,
                                              uint32_t vpt) {
  AlwaysGo go;
  move_tile<false>(src, dst, n_out, op, n_tiles, tile, vpt, go);
}
__device__ __forceinline__ bool op_narrows(uint32_t op) { return op == OP_F2H || op == OP_F2B; }

// ------------------------------------------------------------------------------------------------
// move_kernel: CTAs [0, n_tiles) each take one tile of a large payload; the CTAs after them take the
// small items (header fragments, small payloads), one warp per item.
// ------------------------------------------------------------------------------------------------
struct GuardMid {   // the guarded move: the tile's loads are in flight while the record's guard word arrives; nothing is stored on 0
  uint32_t g;
  __device__ __forceinline__ bool operator()() const { return g != 0; }
};

template <bool GUARD>
__device__ __forceinline__ void move_body(const uint8_t* plan) {
  const PlanHeader& ph = *reinterpret_cast<const PlanHeader*>(plan);
  const uint32_t b = blockIdx.x;
  if (b < ph.n_tiles) {
    uint32_t item, tile;
    if (ph.uniform_tpi) { item = b / ph.uniform_tpi; tile = b - item * ph.uniform_tpi; }
    else {
      const TileRef tr = reinterpret_cast<const TileRef*>(plan + ph.off_tiles)[b];
      item = tr.item; tile = tr.tile;
    }
    const MoveItem& it = reinterpret_cast<const MoveItem*>(plan + ph.off_items)[item];
    if (GUARD) {
      GuardMid mid{ph.guard[item / ph.guard_div]};
      if (it.gstride) { if (mid()) move_tile_gather(SrcView{it.src, it.glen, it.gstride}, it.dst, it.n_out, it.op, it.n_tiles, tile, ph.vec_per_tile); return; }
      move_tile<false>(it.src, it.dst, it.n_out, it.op, it.n_tiles, tile, ph.vec_per_tile, mid);
      return;
    }
    if (it.gstride) { move_tile_gather(SrcView{it.src, it.glen, it.gstride}, it.dst, it.n_out, it.op, it.n_tiles, tile, ph.vec_per_tile); return; }
    AlwaysGo go;
    move_tile<false>(it.src, it.dst, it.n_out, it.op, it.n_tiles, tile, ph.vec_per_tile, go);
  } else {
    const uint32_t warps = blockDim.x >> 5;
    const uint32_t idx = (b - ph.n_tiles) * warps + (threadIdx.x >> 5);
    if (idx >= ph.n_small) return;
    const SmallItem si = reinterpret_cast<const SmallItem*>(plan + ph.off_small)[idx];
    const uint32_t op = si.op & ~OP_FLAG_BLOB;
    const SrcView src{(si.op & OP_FLAG_BLOB) ? plan + si.src : reinterpret_cast<const uint8_t*>(si.src), si.glen, si.gstride};
    const uint32_t lane = threadIdx.x & 31;
    for (uint32_t i = lane; i < si.n_out; i += 32) si.dst[i] = gen_byte(op, src, i);
  }
}

__global__ void __launch_bounds__(kMoveThreads, 3) move_kernel(const uint8_t* __restrict__ plan) {
  pdl_launch_dependents();
  // The plan image was copied by an earlier OPERATION of the stream (complete before the kernel in front of us could start).
  // PlanHeader::independent: that kernel - frame_requests_kernel - writes nothing this plan reads or overwrites (every mover's
  // destination was fixed by the host), so the tiles start while the headers are still being written.
  if (!reinterpret_cast<const PlanHeader*>(plan)->independent) pdl_wait_prior_grids();
  move_body<false>(plan);
}

__global__ void __launch_bounds__(kMoveThreads, 3) move_kernel_inline(const __grid_constant__ InlinePlan plan) {
  pdl_launch_dependents();
  pdl_wait_prior_grids();   // the plan is in the parameters, but sources / the arena may be outputs of earlier kernels
  move_body<false>(plan.bytes);
}

// the same engine over a plan whose items stand for records another kernel vouches for (PlanHeader::guard): the second of the
// three launches of a narrowing batch decode (FusedParams::mode)
__global__ void __launch_bounds__(kMoveThreads, 3) move_guarded_kernel(const uint8_t* __restrict__ plan) {
  pdl_launch_dependents();
  pdl_wait_prior_grids();
  move_body<true>(plan);
}

// ------------------------------------------------------------------------------------------------
// parse kernels (two-phase decode): one lane per record walks the tags into the table
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(32) parse_responses_kernel(const uint8_t* __restrict__ w, const uint64_t* __restrict__ rec_off,
                                                             const uint64_t* __restrict__ rec_len, int n, int max_outputs,
                                                             b200tfs_output* outs, int32_t* n_outs, b200tfs_model_spec* specs,
                                                             int32_t* status, SpillEntry* spill, uint32_t spill_per_rec, uint32_t* spill_used) {
  __shared__ __align__(16) uint8_t lines[32][256];
  int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const uint64_t off = rec_off[r], len = rec_len[r];
  spill_used[r] = 0;
  if (len > 0x7FFFFFFFull) { status[r] = B200TFS_E_PARSE; n_outs[r] = 0; return; }
  Cursor c;
  cur_open(c, w + off, (uint32_t)len, lines[threadIdx.x]);
  SpillArea sp{spill_per_rec ? spill + (size_t)r * spill_per_rec : nullptr, spill_per_rec, 0u};
  int cnt = 0;
  b200tfs_output* mine = outs + (size_t)r * (max_outputs + 1);   // +1: scratch slot
  status[r] = walk_response(c, max_outputs, mine, &cnt, specs + r, sp);
  for (int k = 0; k < cnt; ++k) mine[k].spill_rec = (uint32_t)r;
  n_outs[r] = cnt;
  spill_used[r] = sp.used;
}

__global__ void __launch_bounds__(32) parse_tensors_kernel(const uint8_t* __restrict__ w, const uint64_t* __restrict__ rec_off,
                                                           const uint64_t* __restrict__ rec_len, int n, b200tfs_output* outs,
                                                           int32_t* status, SpillEntry* spill, uint32_t spill_per_rec, uint32_t* spill_used) {
  __shared__ __align__(16) uint8_t lines[32][256];
  int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const uint64_t off = rec_off[r], len = rec_len[r];
  spill_used[r] = 0;
  if (len > 0x7FFFFFFFull) { status[r] = B200TFS_E_PARSE; return; }
  Cursor c;
  cur_open(c, w + off, (uint32_t)len, lines[threadIdx.x]);
  SpillArea sp{spill_per_rec ? spill + (size_t)r * spill_per_rec : nullptr, spill_per_rec, 0u};
  status[r] = walk_tensor_proto(c, outs + r, sp);
  outs[r].spill_rec = (uint32_t)r;
  spill_used[r] = sp.used;
}

// ------------------------------------------------------------------------------------------------
// ------------------------------------------------------------------------------------------------
// staged tile (fused decode, template path): the tile's source bytes are fetched by the TMA engine -
// 1-D bulk copies global -> shared, 32 KB at a time into two buffers, completion on an mbarrier - issued
// BEFORE the template verdict: no register is held across the verdict's barrier (what sank the
// "loads first" variant), and the verdict's DRAM round trip overlaps the tile's.  The CTA then realigns
// from shared memory (two conflict-free 128-bit loads per output vector and a funnel shift - no warp
// shuffles), applies the fix-up and streams the vectors out.
// ------------------------------------------------------------------------------------------------
constexpr uint32_t kStageVecs = kStageVecsHost;             // destination vectors per chunk: 32 KB
constexpr uint32_t kStageBuf = kStageVecs * 16 + 128;       // + the source block after the last vector, rounded
constexpr uint32_t kStageBufs = 2;
constexpr uint32_t kFusedDynSmem = kStageBufs * kStageBuf;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               :: "r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  } while (!ok);
}

struct StagedTile {
  const uint8_t* A;      // 16-byte aligned source address of the tile's first block
  uint8_t* d;            // destination of the tile's first vector (16-byte aligned)
  uint32_t n;            // destination vectors in the tile
  uint32_t k;            // source misalignment: output vector v = bytes [k, k+16) of blocks v, v+1
  uint32_t chunks;       // ceil(n / kStageVecs)
  uint32_t use;          // 0: geometry does not qualify, take move_tile
  uint64_t head, nvec;   // as in move_tile (ragged edges)
};

// geometry of move_tile for the same-width ops, plus the first bulk copies (thread 0)
__device__ __forceinline__ StagedTile staged_begin(const uint8_t* src, uint8_t* dst, uint64_t n_out, uint32_t op, uint32_t tile, uint32_t vpt,
                                                   uint8_t* stage, uint64_t* bars) {
  StagedTile t{};
  if (op != OP_COPY && op != OP_QUIET_DST) return t;
  uint64_t head = (16 - ((uintptr_t)dst & 15)) & 15;
  if (head > n_out) head = n_out;
  if (op == OP_QUIET_DST && (head & 3)) return t;
  const uint8_t* src_body = src + head;
  const uint32_t k = (uint32_t)((uintptr_t)src_body & 15);
  uint64_t nvec = (n_out - head) >> 4;
  if (k) {  // block v+1 is read as well: keep it inside the source
    const uint64_t blocks = (uint64_t)((src + n_out) - (src_body - k)) >> 4;
    const uint64_t lim = blocks ? blocks - 1 : 0;
    if (nvec > lim) nvec = lim;
  }
  t.head = head; t.nvec = nvec; t.k = k; t.use = 1;
  const uint64_t v0 = (uint64_t)tile * vpt;
  t.n = v0 < nvec ? (uint32_t)min((uint64_t)vpt, nvec - v0) : 0u;
  t.A = src_body - k + 16 * v0;
  t.d = dst + head + 16 * v0;
  t.chunks = (t.n + kStageVecs - 1) / kStageVecs;
  if (threadIdx.x == 0) {
    for (uint32_t c = 0; c < min(t.chunks, kStageBufs); ++c) {
      const uint32_t nc = min(kStageVecs, t.n - c * kStageVecs), bytes = 16u * (nc + (k ? 1u : 0u));
      mbar_expect_tx(&bars[c], bytes);
      bulk_g2s(stage + c * kStageBuf, t.A + (uint64_t)c * kStageVecs * 16, bytes, &bars[c]);
    }
  }
  return t;
}

template <uint32_t OP, int Q>
__device__ __forceinline__ void staged_chunk(const uint8_t* buf, uint8_t* dst, uint32_t nc, uint32_t s) {
  const uint4* b = reinterpret_cast<const uint4*>(buf);
  constexpr uint32_t kPer = 1;
  for (uint32_t base = 0; base < nc; base += kPer * kMoveThreads) {
    uint4 lo[kPer], hi[kPer];
#pragma unroll
    for (uint32_t i = 0; i < kPer; ++i) {
      const uint32_t v = base + i * kMoveThreads + threadIdx.x;
      if (v < nc) { lo[i] = b[v]; if (Q >= 0) hi[i] = b[v + 1]; }
    }
#pragma unroll
    for (uint32_t i = 0; i < kPer; ++i) {
      const uint32_t v = base + i * kMoveThreads + threadIdx.x;
      if (v < nc) {
        uint4 o = lo[i];
        if (Q >= 0) o = shift_pair<(Q >= 0 ? Q : 0)>(lo[i], hi[i], s);
        st_stream(dst + 16ull * v, fix_vec<OP>(o));
      }
    }
  }
}

template <uint32_t OP>
__device__ __forceinline__ void staged_chunk_op(const uint8_t* buf, uint8_t* dst, uint32_t nc, uint32_t k) {
  const uint32_t s = (k & 3) * 8;
  if (k == 0) { staged_chunk<OP, -1>(buf, dst, nc, 0); return; }
  switch (k >> 2) {  // uniform across the CTA
    case 0: staged_chunk<OP, 0>(buf, dst, nc, s); break;
    case 1: staged_chunk<OP, 1>(buf, dst, nc, s); break;
    case 2: staged_chunk<OP, 2>(buf, dst, nc, s); break;
    default: staged_chunk<OP, 3>(buf, dst, nc, s); break;
  }
}

// the copies that are in flight must land before their buffers (or the CTA) go away
__device__ __forceinline__ void staged_drain(const StagedTile& t, uint64_t* bars, uint32_t from_chunk) {
  if (!t.use) return;
  for (uint32_t c = from_chunk; c < min(t.chunks, from_chunk + kStageBufs); ++c) mbar_wait(&bars[c % kStageBufs], (c / kStageBufs) & 1);
}

__device__ __forceinline__ void staged_finish(const StagedTile& t, const uint8_t* src, uint8_t* dst, uint64_t n_out, uint32_t op, uint32_t n_tiles,
                                              uint32_t tile, uint8_t* stage, uint64_t* bars) {
  for (uint32_t c = 0; c < t.chunks; ++c) {
    const uint32_t buf = c % kStageBufs, nc = min(kStageVecs, t.n - c * kStageVecs);
    mbar_wait(&bars[buf], (c / kStageBufs) & 1);
    uint8_t* d = t.d + (uint64_t)c * kStageVecs * 16;
    if (op == OP_COPY) staged_chunk_op<OP_COPY>(stage + buf * kStageBuf, d, nc, t.k);
    else staged_chunk_op<OP_QUIET_DST>(stage + buf * kStageBuf, d, nc, t.k);
    if (c + kStageBufs < t.chunks) {   // refill this buffer with the chunk two ahead, once every thread has read it
      __syncthreads();
      if (threadIdx.x == 0) {
        const uint32_t c2 = c + kStageBufs, n2 = min(kStageVecs, t.n - c2 * kStageVecs), bytes = 16u * (n2 + (t.k ? 1u : 0u));
        mbar_expect_tx(&bars[buf], bytes);
        bulk_g2s(stage + buf * kStageBuf, t.A + (uint64_t)c2 * kStageVecs * 16, bytes, &bars[buf]);
      }
    }
  }
  // ragged edges, element-exact (as move_tile)
  if (tile == 0) for (uint64_t i = threadIdx.x; i < t.head; i += blockDim.x) dst[i] = gen_byte(op, src, i);
  if (tile + 1 == n_tiles) for (uint64_t i = t.head + (t.nvec << 4) + threadIdx.x; i < n_out; i += blockDim.x) dst[i] = gen_byte(op, src, i);
}

// decode_fused_kernel: the whole PredictResponse decode in ONE launch.  CTA b belongs to record r with
// local tile j.
//
// Fast path - framing template.  In steady state every response of a model has the same framing
// (same keys, dtypes, dims => the same non-payload bytes at the same offsets).  The previous launch
// left a template of record 0: its framing bytes, where the value chunks lie, and the finished table.
// Each CTA checks, one byte per thread, that this record's framing bytes equal the template's (and
// that packed-varint chunks still end on a terminator); identical framing bytes of an identical
// length parse identically, so the CTA takes its tile straight from the template.  Cost: one DRAM
// round trip for the two framing lines instead of a serial tag walk (a lone GPU lane walks ~100 header
// bytes through many dependent loads).
//
// Slow path - thread 0 walks the tags through the line cache (walker.h), lays the outputs out in the
// record's destination slot and finds which value chunk tile j falls in; CTA (record 0, tile 0) also
// writes the template for the next launch.  CTA j == 0 of every record publishes the table.
// ------------------------------------------------------------------------------------------------
struct FusedJob { const uint8_t* src; uint8_t* dst; uint64_t n_out; uint32_t op, n_tiles, tile, valid, glen, gstride; };

__device__ __forceinline__ void publish_words(void* dst, const void* src, uint32_t bytes) {
  const uint64_t* s = reinterpret_cast<const uint64_t*>(src);
  uint64_t* d = reinterpret_cast<uint64_t*>(dst);
  for (uint32_t i = threadIdx.x; i < bytes / 8; i += blockDim.x) d[i] = s[i];
}

// the serial walk, kept out of line so the fast path's registers stay lean (thread 0 only).  `publish`: this CTA writes the
// record's table (the CTA with j == 0 on the walk path; the record's last CTA when it could not vouch for the template's table)
__device__ __noinline__ void fused_slow_path(const FusedParams& fp, uint32_t r, uint32_t j, uint32_t budget, bool publish, const uint8_t* rec,
                                             uint64_t len, uint8_t* dst_slot, uint8_t* lines, b200tfs_output* outs_s, b200tfs_model_spec& spec_s,
                                             FusedJob& job) {
    int cnt = 0, st;
    Cursor c;
    job.valid = 0;
    if (len > 0x7FFFFFFFull) st = B200TFS_E_PARSE;
    else {
      cur_open(c, rec, (uint32_t)len, lines);
      SpillArea sp{nullptr, 0u, 0u};   // no spill area behind the single-launch decode: such a record is left to the two-phase calls
      st = walk_response(c, kFusedMaxOutputs, outs_s, &cnt, &spec_s, sp);
      if (st == B200TFS_E_SPILL) st = B200TFS_E_NONCANONICAL;
    }
    uint64_t cursor = 0;   // bytes used in this record's destination slot
    uint32_t t_base = 0;   // tiles consumed by earlier chunks
    if (st == B200TFS_OK) {
      cursor = tpl_layout_outputs(outs_s, cnt, fp.dst_stride, fp.cast, fp.varints);
      // tiles are handed out by ascending wire offset of the chunk (same order the template uses)
      uint32_t done_mask[kFusedMaxOutputs] = {0};
      for (;;) {
        int bk = -1, bq = -1; uint64_t best = ~0ull;
        for (int k = 0; k < cnt; ++k) {
          const b200tfs_output& o = outs_s[k];
          if (o.status != B200TFS_OK || !o.n_elems || dtype_info(o.dtype).kind != VK_FIXED) continue;
          for (int q = 0; q < o.n_runs; ++q)
            if (!(done_mask[k] >> q & 1) && o.runs[q].off < best) { best = o.runs[q].off; bk = k; bq = q; }
        }
        if (bk < 0) break;
        done_mask[bk] |= 1u << bq;
        const b200tfs_output& o = outs_s[bk];
        uint64_t run = 0;
        for (int q = 0; q < bq; ++q) run += (uint64_t)o.runs[q].len * o.runs[q].count;
        const b200tfs_run& rn = o.runs[bq];
        const bool narrow = tpl_narrows(fp.cast, o.dtype);
        const uint64_t bytes = ((uint64_t)rn.len * rn.count) >> (narrow ? 1 : 0);     // bytes written
        const uint32_t nt = tiles_for(bytes, fp.vpt);
        if (j >= t_base && j < t_base + nt) {
          job.src = rec + rn.off; job.dst = dst_slot + o.dst_off + (narrow ? run / 2 : run); job.n_out = bytes;
          job.op = tpl_move_op(fp.cast, o.dtype); job.n_tiles = nt; job.tile = j - t_base; job.valid = 1;
          job.glen = rn.count > 1 ? rn.len : 0u; job.gstride = rn.count > 1 ? rn.stride : 0u;   // a row of unpacked elements: gathered
        }
        t_base += nt;
      }
      if (t_base > budget) st = B200TFS_E_NONCANONICAL;  // more chunks than the launch budgeted tiles for
    }
    if (publish) {
      if (fp.stats) atomicAdd(&fp.stats[2], 1ull);
      fp.status[r] = st;
      fp.n_outs[r] = (st == B200TFS_OK) ? cnt : 0;
      fp.specs[r] = spec_s;
      for (int k = 0; k < cnt && st == B200TFS_OK; ++k) fp.outs[(size_t)r * kFusedMaxOutputs + k] = outs_s[k];
      if (r == 0) {   // leave the template for the next launch, and its inline part in pinned memory for the host
        if (len <= 0x7FFFFFFFull) tpl_learn(fp.tpl_write, c, (uint32_t)len, outs_s, cnt, spec_s, st, fp.vpt, (cursor + 255) & ~255ull, fp.serial, fp.cast,
                                            fp.varints);
        else fp.tpl_write->in.head.valid = 0;
        if (fp.tpl_pinned) {   // valid or not, stamped with this launch's serial: the host drops what it knew before either way
          fp.tpl_pinned->head.valid = 0;
          __threadfence_system();
          const uint64_t* s8 = reinterpret_cast<const uint64_t*>(&fp.tpl_write->in);
          uint64_t* d8 = reinterpret_cast<uint64_t*>(fp.tpl_pinned);
          const bool ok = fp.tpl_write->in.head.valid != 0;
          if (ok) for (uint32_t q = sizeof(TplHead) / 8; q < sizeof(TplInline) / 8; ++q) d8[q] = s8[q];
          __threadfence_system();
          TplHead h = fp.tpl_write->in.head;
          h.serial = fp.serial; h.valid = ok ? 1u : 0u;
          const uint64_t* h8 = reinterpret_cast<const uint64_t*>(&h);
          for (uint32_t q = sizeof(TplHead) / 8; q-- > 0;) d8[q] = h8[q];   // the word with the valid flag (the first) last
        }
      }
    }
    if (st != B200TFS_OK) job.valid = 0;
}

// decode_fused_kernel: the whole PredictResponse decode in ONE launch.  CTA b belongs to record r with local tile j.
//
// Framing template (tpl.h).  In steady state every response of a model has the same framing (same keys, dtypes, dims => the
// same non-payload bytes at the same offsets).  The template rides in the kernel parameters when the host has it (it walked
// record 0 itself, or found the previous launch's template in pinned memory with the stream idle): the CTA issues its tile's
// loads at once and checks, one byte per thread, that this record's framing bytes equal the template's while those loads are
// in flight (packed-varint chunks must still end on a terminator) - one DRAM round trip in all.  Otherwise the template the
// previous launch left in device memory is used (one more dependent load).  A record that misses the template is walked:
// thread 0 goes through the tags with the line cache (a lone GPU lane walks ~100 header bytes through dependent loads), lays the outputs out
// and finds which value chunk tile j falls in; CTA (record 0, tile 0) also leaves the template for the next launch.
//
// STAGED: tiles of more than one 32 KB chunk (big batches) take the TMA-staged path above; the other instantiation - a single
// response, small batches - carries none of that code and instead runs the verdict as the `mid` hook of the tile move (the
// registers that holds across the barrier cost the big-batch kernel a CTA per SM, so only this one does it).
// CAST: the instantiations behind b200tfs_set_decode_cast carry the narrowing tile move as well; the plain ones are exactly the
// round-1/2 kernels (the extra branch and registers slowed the single-response launch when it lived in the same kernel).
template <bool STAGED, bool CAST>
__device__ __forceinline__ void decode_fused_body(const FusedParams& fp) {
  pdl_launch_dependents();
  __shared__ __align__(16) uint8_t lines[256];
  __shared__ b200tfs_output outs_s[kFusedMaxOutputs + 1];  // +1: scratch slot for an entry whose key repeats
  __shared__ b200tfs_model_spec spec_s;
  __shared__ FusedJob job;
  extern __shared__ __align__(128) uint8_t stage_smem[];     // STAGED: kFusedDynSmem bytes, the staged tile's two buffers
  __shared__ __align__(8) uint64_t stage_bars[kStageBufs];
  __shared__ TplChunk ch_s[kTplChunks];
  __shared__ TplHead th_s;
  if (STAGED && threadIdx.x == 0) {   // made visible by the template staging's barrier
    for (uint32_t q = 0; q < kStageBufs; ++q) mbar_init(&stage_bars[q], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  const uint32_t b = blockIdx.x + fp.tile_bias;
  uint32_t r, j, budget;
  uint64_t off, len;
  if (fp.n <= kFusedInlineRecs) {
    r = 0;
    while (r + 1 < (uint32_t)fp.n && b >= fp.inl.tile_start[r + 1]) ++r;
    j = b - fp.inl.tile_start[r]; off = fp.inl.off[r]; len = fp.inl.len[r];
    budget = fp.inl.tile_start[r + 1] - fp.inl.tile_start[r];
  } else {
    r = fp.cta_rec[b];
    const uint32_t t0 = fp.tile_start[r];
    j = b - t0; off = fp.rec_off[r]; len = fp.rec_len[r];
    budget = fp.tile_start[r + 1] - t0;
  }
  const uint8_t* rec = fp.w + off;
  uint8_t* dst_slot = fp.dst + (uint64_t)r * fp.dst_stride;
  pdl_wait_prior_grids();   // the template was written by the previous decode launch; the wire may be fresh too
  if (CAST && fp.mode == 2 && fp.guard[r] != 0) return;    // verified and moved by the two launches before this one

  // One template per launch: the one in the kernel parameters when the host supplied it, else the one the previous launch left
  // in device memory.  (Trying both in turn kept too much state alive across the tile move: 500-700 bytes of spills.)  A record
  // that misses it is walked; record 0's walk leaves the new template in device AND pinned memory, where the host finds it.
  const Template* T = fp.tpl_read;
  const bool inl = !STAGED && fp.tpli.head.valid != 0;   // the batch kernel hides the template load behind its bulk copies: no gain, and 80 bytes of spills
  uint32_t live = budget;   // CTAs of this record able to take a tile, should the walk be needed
  const uint32_t i = threadIdx.x;
  {
    if (inl) {
      if (i < kTplChunks) ch_s[i] = fp.tpli.chunk[i];
      if (i == kTplChunks) th_s = fp.tpli.head;
    } else {
      // five threads stage the header and chunk table (independent loads: one L2 round trip).  (An earlier version kept the
      // chunk table in a per-thread array: it landed in local memory, 32 KB of extra DRAM traffic per CTA.)
      if (i < kTplChunks) ch_s[i] = T->in.chunk[i];
      if (i == kTplChunks) th_s = T->in.head;
    }
    __syncthreads();
    const uint32_t nch = th_s.n_chunks;
    if (th_s.valid && th_s.rec_len == len && th_s.vpt == fp.vpt && th_s.cast == fp.cast && th_s.varints == fp.varints && th_s.dst_need <= fp.dst_stride &&
        (th_s.total_tiles < budget || (CAST && fp.mode == 1))) {
      // The verdict: do this record's framing bytes equal the template's (and do packed-varint chunks still end on a terminator)?
      // It needs the record's framing bytes - a DRAM round trip.  The batch kernel decides per CTA (one byte per thread, one
      // barrier).  The single-response kernel decides per WARP - every warp compares all framing bytes itself (same bytes, same
      // answer) - so that no CTA-wide barrier sits between a warp's loads and its stores: a warp whose tile data has arrived
      // stores it while other warps' loads are still in flight, as in the plain move.
      auto verdict = [&]() -> bool {
        bool same = true;
        if (!STAGED && fp.trusted && inl) return true;
        if (STAGED) {
          if (i < th_s.framing_len) {
            uint32_t w = i;
            for (uint32_t q = 0; q < nch; ++q) if (ch_s[q].fpos <= i) w += ch_s[q].len;
            same = rec[w] == T->in.framing[i];
          }
          if (i < nch && ch_s[i].is_varint && ch_s[i].len) same = same && !(rec[ch_s[i].wire_off + ch_s[i].len - 1] & 0x80);
          return __syncthreads_and(same) != 0;
        }
        const uint32_t lane = i & 31;
        for (uint32_t k = lane; k < th_s.framing_len; k += 32) {
          uint32_t w = k;
          for (uint32_t q = 0; q < nch; ++q) if (ch_s[q].fpos <= k) w += ch_s[q].len;
          const uint8_t want = inl ? fp.tpli.framing[k] : T->in.framing[k];
          same = same && rec[w] == want;
        }
        if (lane < nch && ch_s[lane].is_varint && ch_s[lane].len) same = same && !(rec[ch_s[lane].wire_off + ch_s[lane].len - 1] & 0x80);
        return __all_sync(0xFFFFFFFFu, same) != 0;
      };
      uint32_t t_base = 0, mine = kTplChunks;
      for (uint32_t q = 0; q < nch; ++q) {
        const uint32_t nt = ch_s[q].n_tiles;
        if (j >= t_base && j < t_base + nt) { mine = q; break; }
        t_base += nt;
      }
      if (CAST && fp.mode == 1) {   // verify only: CTA 0 answers in the record's guard word, CTA 1 (the last) publishes the table
        mine = kTplChunks;
        const bool ok = verdict();
        if (j == 0) { if (threadIdx.x == 0) fp.guard[r] = ok ? 1u : 0u; return; }
        if (!ok) return;
      }
      // A slack CTA (the launch budgets kFusedSlackTiles more CTAs per record than tiles_for(len), for records whose
      // values lie in several chunks) has nothing to do when the record carries the template's framing - and 8 of the 11
      // CTAs of a 602 KB record are slack: leave now, before the verdict's round trip.  Should the record fail the
      // verdict after all, the CTAs that stayed walk it; if it then needs more tiles than stayed, its status says so.
      if (mine == kTplChunks && j != 0 && j != budget - 1) return;
      live = max(th_s.total_tiles, 1u);
      bool hit;
      if (STAGED) {
        // the tile's bytes start moving now (TMA bulk copies into shared memory), the verdict's round trip overlaps theirs
        StagedTile stg{};
        const bool narrow = CAST && mine < kTplChunks && op_narrows(ch_s[mine].op);
        if (mine < kTplChunks && !narrow)
          stg = staged_begin(rec + ch_s[mine].wire_off, dst_slot + ch_s[mine].dst_off, ch_s[mine].len, ch_s[mine].op, j - t_base, fp.vpt,
                             stage_smem, stage_bars);
        if (narrow)   // the general tile move with the verdict between its first loads and its first stores (CTA-uniform: a barrier inside)
          hit = move_tile<false>(rec + ch_s[mine].wire_off, dst_slot + ch_s[mine].dst_off, (uint64_t)(ch_s[mine].len >> 1), ch_s[mine].op,
                                 ch_s[mine].n_tiles, j - t_base, fp.vpt, verdict);
        else hit = verdict();
        if (hit && mine < kTplChunks && !narrow) {
          if (stg.use)
            staged_finish(stg, rec + ch_s[mine].wire_off, dst_slot + ch_s[mine].dst_off, ch_s[mine].len, ch_s[mine].op, ch_s[mine].n_tiles,
                          j - t_base, stage_smem, stage_bars);
          else
            move_tile_cold(rec + ch_s[mine].wire_off, dst_slot + ch_s[mine].dst_off, ch_s[mine].len, ch_s[mine].op, ch_s[mine].n_tiles, j - t_base,
                           fp.vpt);
        }
        if (!hit) staged_drain(stg, stage_bars, 0);   // let the copies land, then walk the record
      } else if (CAST && mine < kTplChunks && op_narrows(ch_s[mine].op)) {
        // narrowing tile: its loads go out first as well (general tile move, inlined into the cast instantiations only)
        hit = move_tile<false>(rec + ch_s[mine].wire_off, dst_slot + ch_s[mine].dst_off, (uint64_t)(ch_s[mine].len >> 1), ch_s[mine].op,
                               ch_s[mine].n_tiles, j - t_base, fp.vpt, verdict);
      } else if (mine < kTplChunks) {
        // the tile's loads go out first; the verdict runs while they are in flight and decides whether anything is stored
        hit = move_tile<true>(rec + ch_s[mine].wire_off, dst_slot + ch_s[mine].dst_off, ch_s[mine].len, ch_s[mine].op, ch_s[mine].n_tiles,
                              j - t_base, fp.vpt, verdict);
      } else hit = verdict();
      if (hit) {
        if (j == budget - 1) {   // the record's last CTA - a slack CTA with no tile - publishes the table, so no tile waits on it
          // the table entries live in the device template; an inline template vouches for them only if both carry the same serial
          const bool table_ok = !inl || (T->in.head.valid && T->in.head.serial == th_s.serial);
          if (table_ok) {
            if (threadIdx.x == 0 && fp.stats) atomicAdd(&fp.stats[inl ? 0 : 1], 1ull);
            publish_words(fp.outs + (size_t)r * kFusedMaxOutputs, T->outs, th_s.n_outs * (uint32_t)sizeof(b200tfs_output));
            publish_words(fp.specs + r, &T->spec, (uint32_t)sizeof(b200tfs_model_spec));
            if (threadIdx.x == 0) { fp.status[r] = B200TFS_OK; fp.n_outs[r] = (int32_t)th_s.n_outs; }
            // hand the template on to the next launch (launches alternate between the two slots).  Unconditionally: the warps
            // of this CTA are not in step (per-warp verdict), and a test of the target slot ("does it hold this template
            // already?") read the words the faster warps had just written - the slower ones then skipped their share of the
            // copy and left a torn template behind (found by compute-sanitizer's slow motion, never seen at full speed).
            if (r == 0) publish_words(fp.tpl_write, T, (uint32_t)sizeof(Template));
          } else if (threadIdx.x == 0) {
            fused_slow_path(fp, r, 0, budget, true, rec, len, dst_slot, lines, outs_s, spec_s, job);   // walk for the table only
          }
        }
        return;
      }
    }
  }

  // ---- the walk: thread 0 goes through the tags ----
  if (CAST && fp.mode == 1) { if (j == 0 && threadIdx.x == 0) fp.guard[r] = 0u; return; }   // left to the third launch
  if (threadIdx.x == 0) fused_slow_path(fp, r, j, live, j == 0, rec, len, dst_slot, lines, outs_s, spec_s, job);
  __syncthreads();
  if (job.valid) {
    if (job.gstride) move_tile_gather(SrcView{job.src, job.glen, job.gstride}, job.dst, job.n_out, job.op, job.n_tiles, job.tile, fp.vpt);
    else if (CAST && op_narrows(job.op)) move_tile_narrow(job.src, job.dst, job.n_out, job.op, job.n_tiles, job.tile, fp.vpt);
    else move_tile_cold(job.src, job.dst, job.n_out, job.op, job.n_tiles, job.tile, fp.vpt);
  }
}

// two CTAs per SM: the tile (8 x 128-bit per thread) stays in registers across the verdict's barrier without spilling; this instantiation serves
// single responses and small batches, where a third resident CTA has nothing to hide
__global__ void __launch_bounds__(kMoveThreads, 2) decode_fused_kernel(const __grid_constant__ FusedParams fp) { decode_fused_body<false, false>(fp); }
// the staged (batch) instantiations too: on sm_90a a third CTA per SM caps them at 80 registers and spills the walker's state
// (132 B of stores); at two the batch decode measured 3-4 % faster on an H100 (C2 773 -> 750 us, C5 share 3569 -> 3426 us)
__global__ void __launch_bounds__(kMoveThreads, 2) decode_fused_staged_kernel(const __grid_constant__ FusedParams fp) { decode_fused_body<true, false>(fp); }
__global__ void __launch_bounds__(kMoveThreads, 2) decode_fused_cast_kernel(const __grid_constant__ FusedParams fp) { decode_fused_body<false, true>(fp); }
__global__ void __launch_bounds__(kMoveThreads, 2) decode_fused_staged_cast_kernel(const __grid_constant__ FusedParams fp) { decode_fused_body<true, true>(fp); }

// ------------------------------------------------------------------------------------------------
// packed varints: venc_len / venc_emit / vdec_count / vdec_emit
// ------------------------------------------------------------------------------------------------
#include "varint_kernels.cuh"

// ------------------------------------------------------------------------------------------------
// concat_plan_kernel (plan.h ConcatPlan): one CTA plans b200tfs_decode_concat.  Per requested key, pass A matches the key in
// every record's table and finds the first record that decoded it (the reference for dtype, rank and trailing dims); pass B
// checks every record against it, scans the bytes of the records into offsets inside the key's destination and the move
// tiles into the tile table, and writes the move items and the varint table.  Block scans with the carry in a register:
// nothing waits on another CTA, and a replayed graph re-plans from whatever row counts the new records carry.
// ------------------------------------------------------------------------------------------------
// exclusive scan of one value per thread across the CTA; `carry` (uniform) advances by the round's total
__device__ __forceinline__ uint64_t concat_scan(uint64_t v, uint64_t& carry, unsigned long long* warp_sum) {
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  uint64_t inc = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint64_t x = __shfl_up_sync(0xFFFFFFFFu, inc, d);
    if (lane >= (uint32_t)d) inc += x;
  }
  if (lane == 31) warp_sum[wid] = inc;
  __syncthreads();
  uint64_t before = carry, round = 0;
  for (uint32_t w = 0; w < kConcatPlanThreads / 32; ++w) {
    const uint64_t x = warp_sum[w];
    if (w < wid) before += x;
    round += x;
  }
  __syncthreads();
  carry += round;
  return before + inc - v;
}

// pass A of the key plans (concat_plan_kernel, padded_plan_kernel): the key in each record's table, and the record's own verdict
// on it, into cp.kst / cp.match; *ref_rec (shared, n on entry) receives the first record that decoded the key
__device__ __forceinline__ void plan_match_key(const ConcatPlan& cp, const uint8_t* kb, uint32_t key_len, uint32_t k, uint32_t* ref_rec) {
  const uint32_t n = cp.n, nk = cp.n_keys;
  for (uint32_t r = threadIdx.x; r < n; r += kConcatPlanThreads) {
    int32_t st = cp.rec_status[r], m = -1;
    if (st == B200TFS_E_SPILL || st == B200TFS_E_SIZE) st = B200TFS_E_NONCANONICAL;   // more than the table holds: another route
    if (st == B200TFS_OK) {
      const b200tfs_output* t = cp.outs + (size_t)r * cp.out_stride;
      const uint8_t* rec = cp.w + cp.rec_off[r];
      for (int32_t j = 0; j < cp.n_outs[r] && m < 0; ++j) {
        if (t[j].key_len != key_len) continue;
        bool same = true;
        for (uint32_t i = 0; i < key_len && same; ++i) same = rec[t[j].key_off + i] == kb[i];
        if (same) m = j;
      }
      if (m < 0) st = B200TFS_E_KEY;
      else {
        const b200tfs_output& o = t[m];
        st = o.status;
        if (st == B200TFS_OK && o.rank == 0) st = B200TFS_E_SHAPE;
        if (st == B200TFS_OK && o.rank > B200TFS_MAX_RANK) st = B200TFS_E_NONCANONICAL;
      }
    }
    cp.kst[(size_t)r * nk + k] = st;
    cp.match[(size_t)r * nk + k] = m;
    if (st == B200TFS_OK) atomicMin(ref_rec, r);
  }
}

// pass A of key k, called by every thread of the CTA (`ref_rec`: shared scratch): the output of the first record that decoded the
// key, the reference of pass B, or nullptr when no record did
__device__ __forceinline__ const b200tfs_output* plan_key_reference(const ConcatPlan& cp, const uint8_t* kb, uint32_t key_len, uint32_t k,
                                                                    uint32_t* ref_rec) {
  if (threadIdx.x == 0) *ref_rec = cp.n;
  __syncthreads();
  plan_match_key(cp, kb, key_len, k, ref_rec);
  __syncthreads();
  const uint32_t rr = *ref_rec;
  return rr < cp.n ? cp.outs + (size_t)rr * cp.out_stride + cp.match[(size_t)rr * cp.n_keys + k] : nullptr;
}

// kStrings: the DT_STRING outputs get places too (b200tfs_decode_concat_strings): 8 * n_strings bytes of int64 offsets, and one
// more entry behind them, in the key's destination; string_kernels.cuh fills them.  Without it they are left to the host.
template <bool kStrings>
__device__ __forceinline__ void concat_plan_body(const ConcatPlan& cp) {
  __shared__ unsigned long long warp_sum[kConcatPlanThreads / 32];
  __shared__ uint32_t ref_rec;
  const uint32_t n = cp.n, nk = cp.n_keys;
  const uint64_t n_items = (uint64_t)n * nk * B200TFS_MAX_RUNS;
  const PlanGeometry g = plan_geometry(n_items, 0, 0);   // tile refs run from off_tiles to the end of the image; no small items
  MoveItem* items = reinterpret_cast<MoveItem*>(cp.plan + g.off_items);
  TileRef* tref = reinterpret_cast<TileRef*>(cp.plan + g.off_tiles);
  uint64_t tile_carry = 0;
  for (uint32_t k = 0; k < nk; ++k) {
    const ConcatKeyDev key = cp.keys[k];
    const b200tfs_output* ro = plan_key_reference(cp, key.key, key.key_len, k, &ref_rec);
    // pass B: consistency, offsets, tiles, items
    uint64_t byte_carry = 0;
    for (uint32_t r0 = 0; r0 < n; r0 += kConcatPlanThreads) {      // uniform trip count: the scans have barriers inside
      const uint32_t r = r0 + threadIdx.x;
      int32_t st = B200TFS_E_ARG;
      const b200tfs_output* o = nullptr;
      uint64_t bytes = 0, tail = 0;
      if (r < n) {
        st = cp.kst[(size_t)r * nk + k];
        const int32_t m = cp.match[(size_t)r * nk + k];
        if (m >= 0) o = cp.outs + (size_t)r * cp.out_stride + m;
        if (st == B200TFS_OK) {
          if (o->dtype != ro->dtype) st = B200TFS_E_DTYPE;
          else if (o->rank != ro->rank) st = B200TFS_E_SHAPE;
          else for (int32_t d = 1; d < o->rank; ++d) if (o->dims[d] != ro->dims[d]) st = B200TFS_E_SHAPE;
        }
        const bool str = st == B200TFS_OK && dtype_info(o->dtype).kind == VK_STRING;
        if (str && !kStrings) st = B200TFS_E_NONCANONICAL;   // strings are decoded on the host
        if (st == B200TFS_OK) bytes = str ? 8 * o->n_strings : tpl_narrows(cp.cast, o->dtype) ? o->n_elems * 2 : o->dst_bytes;
        if (kStrings && str) tail = 8;                       // the entry behind the record's last string
      }
      const uint64_t off = concat_scan(bytes, byte_carry, warp_sum);
      if (st == B200TFS_OK && off + bytes + tail > key.cap) st = B200TFS_E_SIZE;
      uint32_t tiles = 0;
      const bool narrow = st == B200TFS_OK && tpl_narrows(cp.cast, o->dtype);
      if (st == B200TFS_OK && bytes && dtype_info(o->dtype).kind == VK_FIXED)   // OK fixed-width outputs with elements have value runs
        for (int32_t q = 0; q < o->n_runs; ++q) tiles += tiles_for(((uint64_t)o->runs[q].len * o->runs[q].count) >> (narrow ? 1 : 0), cp.vpt);
      const uint64_t first = concat_scan(tiles, tile_carry, warp_sum);
      if (r < n) {
        if (tiles && first + tiles > cp.tile_cap) st = B200TFS_E_NONCANONICAL;   // past the host's bound (never: concat_record_tile_bound)
        if (st == B200TFS_OK && tiles) {
          const uint8_t* rec = cp.w + cp.rec_off[r];
          const uint32_t op = tpl_move_op(cp.cast, o->dtype);
          uint64_t t = first, run = 0;
          for (int32_t q = 0; q < o->n_runs; ++q) {
            const b200tfs_run& rn = o->runs[q];
            const uint64_t nb = ((uint64_t)rn.len * rn.count) >> (narrow ? 1 : 0);
            const uint32_t nt = tiles_for(nb, cp.vpt), item = (uint32_t)(((uint64_t)r * nk + k) * B200TFS_MAX_RUNS + q);
            items[item] = MoveItem{rec + rn.off, key.dst + off + run, nb, op, nt, rn.count > 1 ? rn.len : 0u, rn.count > 1 ? rn.stride : 0u};
            for (uint32_t i = 0; i < nt && t + i < cp.tile_cap; ++i) tref[t + i] = TileRef{item, i};
            t += nt;
            run += nb;
          }
        }
        b200tfs_output v{};
        if (o) v = *o;
        v.status = st;
        v.dst_off = (uint64_t)(uintptr_t)(key.dst + off);
        v.dst_bytes = bytes;
        cp.vouts[(size_t)r * kFusedMaxOutputs + k] = v;
        if (k == 0) { cp.vn_outs[r] = (int32_t)nk; cp.vrec_status[r] = B200TFS_OK; }
      }
    }
  }
  if (threadIdx.x == 0) {
    PlanHeader ph{};
    ph.n_items = (uint32_t)n_items;
    ph.n_tiles = (uint32_t)min(tile_carry, (uint64_t)cp.tile_cap);
    ph.vec_per_tile = cp.vpt;
    ph.off_items = (uint32_t)g.off_items;
    ph.off_tiles = (uint32_t)g.off_tiles;
    ph.off_small = (uint32_t)g.off_small;
    ph.guard_div = 1;
    *reinterpret_cast<PlanHeader*>(cp.plan) = ph;
  }
}

__global__ void __launch_bounds__(kConcatPlanThreads) concat_plan_kernel(const __grid_constant__ ConcatPlan cp) { concat_plan_body<false>(cp); }
__global__ void __launch_bounds__(kConcatPlanThreads) concat_plan_strings_kernel(const __grid_constant__ ConcatPlan cp) {
  concat_plan_body<true>(cp);
}

// ------------------------------------------------------------------------------------------------
// DT_STRING keys of the concatenated decode: str_index / str_scan / str_copy / str_fix
// ------------------------------------------------------------------------------------------------
#include "string_kernels.cuh"

// ------------------------------------------------------------------------------------------------
// decode into one padded tensor per key: padded_plan_kernel / padded_emit_kernel, and for DT_STRING keys pad_str_index /
// pad_str_scan / pad_str_copy / pad_str_fix
// ------------------------------------------------------------------------------------------------
#include "padded_kernels.cuh"

// ------------------------------------------------------------------------------------------------
// tf.Example requests (Classify / Regress): ex_count / ex_scan / ex_emit / ex_frame
// ------------------------------------------------------------------------------------------------
#include "example_kernels.cuh"

// ------------------------------------------------------------------------------------------------
// Classify / Regress responses: xr_index / xr_scan / xr_emit / xr_compare / xr_publish
// ------------------------------------------------------------------------------------------------
#include "example_resp_kernels.cuh"

// ------------------------------------------------------------------------------------------------
// MultiInference responses: mi_index, then the Classify / Regress kernels per task
// ------------------------------------------------------------------------------------------------
#include "multi_resp_kernels.cuh"

// ------------------------------------------------------------------------------------------------
// PredictRequests cut out of padded tensors: unpad_plan / unpad_len / unpad_layout / unpad_frame / move / unpad_emit
// ------------------------------------------------------------------------------------------------
#include "unpad_kernels.cuh"

// ------------------------------------------------------------------------------------------------
// frame_requests_kernel (plan.h "deferred framing"): one thread per request runs frame_request (framing.h): the framing writers
// count the record from the job totals the counting kernel just produced, the record is placed in its slot (largest payload
// 128-byte aligned, like the host planner's place_record), and a second pass writes every framing byte and patches the
// destinations of the payload movers behind it.
// ------------------------------------------------------------------------------------------------
constexpr uint32_t kFrameThreads = 128;             // requests per CTA (one thread each)

__global__ void __launch_bounds__(kFrameThreads) frame_requests_kernel(const __grid_constant__ FrameTables ft) {
  pdl_launch_dependents();       // an independent move plan (PlanHeader::independent) may start right behind us
  const uint32_t r = blockIdx.x * kFrameThreads + threadIdx.x;
  if (r < ft.n) frame_request(ft, r);
}

cudaError_t launch_frame_requests(const FrameTables& ft, cudaStream_t stream) {
  if (!ft.n) return cudaSuccess;
  frame_requests_kernel<<<(ft.n + kFrameThreads - 1) / kFrameThreads, kFrameThreads, 0, stream>>>(ft);
  return cudaGetLastError();
}

// TensorFlow's MakeNdarray padding (B200TFS_OF_PAD_EDGE): elements [have, n_elems) of dst take the value of element
// have-1, or zero when there is none.  `have` comes from the host (fixed-width values: known from the chunk lengths) or
// from device memory (packed varints: the terminator count the decode kernels just produced).
__global__ void __launch_bounds__(256) fill_edge_kernel(uint8_t* __restrict__ dst, uint32_t elem_size, uint64_t have_imm,
                                                        const unsigned long long* __restrict__ have_dev, uint64_t n_elems) {
  const uint64_t have = have_dev ? (uint64_t)*have_dev : have_imm;
  if (have >= n_elems) return;
  uint8_t last[16];
#pragma unroll
  for (uint32_t b = 0; b < 16; ++b) last[b] = (have && b < elem_size) ? dst[(have - 1) * elem_size + b] : (uint8_t)0;
  for (uint64_t i = have + blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n_elems; i += (uint64_t)gridDim.x * blockDim.x)
#pragma unroll
    for (uint32_t b = 0; b < 16; ++b) if (b < elem_size) dst[i * elem_size + b] = last[b];
}

// ------------------------------------------------------------------------------------------------
// launchers (the only symbols codec_host.cpp sees)
// ------------------------------------------------------------------------------------------------
// launch, optionally with programmatic stream serialization (see pdl_* above).  Measured on the C2 bench:
// with it, overlapping lanes gained a little bandwidth but a single stream of back-to-back launches
// got slower per launch, so it is opt-in: B200TFS_PDL=1.
template <class... KArgs, class... Args>
static cudaError_t launch_pdl(void (*kernel)(KArgs...), uint32_t grid, uint32_t block, uint32_t dyn_smem, cudaStream_t stream, Args&&... args) {
  static const bool env_off = [] { const char* e = getenv("B200TFS_PDL"); return !(e && e[0] == '1'); }();
  const bool off = env_off;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(grid); cfg.blockDim = dim3(block); cfg.dynamicSmemBytes = dyn_smem; cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = off ? 0 : 1;
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

cudaError_t launch_move(const uint8_t* plan_dev, const uint8_t* plan_host, uint32_t plan_bytes, uint32_t n_tiles,
                        uint32_t n_small, cudaStream_t stream) {
  const uint32_t warps = kMoveThreads / 32;
  const uint32_t grid = n_tiles + (n_small + warps - 1) / warps;
  if (grid == 0) return cudaSuccess;
  if (plan_dev == nullptr) {
    InlinePlan ip;
    memcpy(ip.bytes, plan_host, plan_bytes);
    return launch_pdl(move_kernel_inline, grid, kMoveThreads, 0, stream, ip);
  }
  // a plan whose movers need nothing from the kernel in front of them (PlanHeader::independent) is launched with programmatic
  // stream serialization whatever B200TFS_PDL says: overlapping that kernel is the point
  if (!(plan_host && reinterpret_cast<const PlanHeader*>(plan_host)->independent)) return launch_pdl(move_kernel, grid, kMoveThreads, 0, stream, plan_dev);
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(grid); cfg.blockDim = dim3(kMoveThreads); cfg.dynamicSmemBytes = 0; cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, move_kernel, plan_dev);
}

cudaError_t launch_parse_responses(const uint8_t* w, const uint64_t* rec_off, const uint64_t* rec_len, int n, int max_outputs,
                                   b200tfs_output* outs, int32_t* n_outs, b200tfs_model_spec* specs, int32_t* status,
                                   void* spill, uint32_t spill_per_rec, uint32_t* spill_used, cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  parse_responses_kernel<<<(n + 31) / 32, 32, 0, stream>>>(w, rec_off, rec_len, n, max_outputs, outs, n_outs, specs, status,
                                                          (SpillEntry*)spill, spill_per_rec, spill_used);
  return cudaGetLastError();
}

cudaError_t launch_parse_tensors(const uint8_t* w, const uint64_t* rec_off, const uint64_t* rec_len, int n, b200tfs_output* outs,
                                 int32_t* status, void* spill, uint32_t spill_per_rec, uint32_t* spill_used, cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  parse_tensors_kernel<<<(n + 31) / 32, 32, 0, stream>>>(w, rec_off, rec_len, n, outs, status, (SpillEntry*)spill, spill_per_rec, spill_used);
  return cudaGetLastError();
}

uint32_t tiles_for_host(uint64_t n_out, uint32_t vpt) { return tiles_for(n_out, vpt); }

cudaError_t launch_fill_edge(uint8_t* dst, uint32_t elem_size, uint64_t have, const unsigned long long* have_dev, uint64_t n_elems,
                             cudaStream_t stream) {
  if (!n_elems) return cudaSuccess;
  const uint64_t blocks = std::min<uint64_t>((n_elems + 255) / 256, 132 * 8);   // 8 CTAs on each of the H100's 132 SMs
  fill_edge_kernel<<<(uint32_t)blocks, 256, 0, stream>>>(dst, elem_size, have, have_dev, n_elems);
  return cudaGetLastError();
}

cudaError_t launch_decode_fused(const FusedParams& fp, uint32_t grid, cudaStream_t stream) {
  if (!grid) return cudaSuccess;
  {   // the opt-in to > 48 KB of dynamic shared memory is per device (a process may drive several: ShardedCodec)
    static bool opted[64] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) dev = 0;
    if (!opted[dev]) {
      cudaError_t attr = cudaFuncSetAttribute(decode_fused_staged_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFusedDynSmem);
      if (attr == cudaSuccess) attr = cudaFuncSetAttribute(decode_fused_staged_cast_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFusedDynSmem);
      if (attr != cudaSuccess) return attr;
      opted[dev] = true;
    }
  }
  // Tiles of more than one 32 KB chunk (big batches: 64 KB per CTA) go through the TMA-staged path, which moved
  // big batches faster.  One-chunk tiles (a single 4 MiB response) keep the register path and no staging buffers: there
  // the staged path gained little on one stream and lost bandwidth when many lanes overlap.
  if (fp.cast) {
    if (fp.vpt > kStageVecs && fp.mode != 1) return launch_pdl(decode_fused_staged_cast_kernel, grid, kMoveThreads, kFusedDynSmem, stream, fp);
    return launch_pdl(decode_fused_cast_kernel, grid, kMoveThreads, 0, stream, fp);
  }
  if (fp.vpt > kStageVecs) return launch_pdl(decode_fused_staged_kernel, grid, kMoveThreads, kFusedDynSmem, stream, fp);
  return launch_pdl(decode_fused_kernel, grid, kMoveThreads, 0, stream, fp);
}

cudaError_t launch_concat_plan(const ConcatPlan& cp, uint32_t move_grid, cudaStream_t stream, bool strings) {
  if (strings) concat_plan_strings_kernel<<<1, kConcatPlanThreads, 0, stream>>>(cp);
  else concat_plan_kernel<<<1, kConcatPlanThreads, 0, stream>>>(cp);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess || !move_grid) return e;
  // a plain launch: move_kernel reads PlanHeader::independent before it waits on the kernel in front of it, and here that kernel
  // writes the header
  move_kernel<<<move_grid, kMoveThreads, 0, stream>>>((const uint8_t*)cp.plan);
  return cudaGetLastError();
}

cudaError_t launch_move_guarded(const uint8_t* plan_dev, uint32_t n_tiles, cudaStream_t stream) {
  if (!n_tiles) return cudaSuccess;
  return launch_pdl(move_guarded_kernel, n_tiles, kMoveThreads, 0, stream, plan_dev);
}

cudaError_t launch_venc_len(const VarTables& tb, cudaStream_t stream) {
  if (!tb.n_tiles) return cudaSuccess;
  venc_len_kernel<<<tb.n_tiles, kVarThreads, 0, stream>>>(tb);
  return cudaGetLastError();
}
cudaError_t launch_venc_emit(const VarTables& tb, cudaStream_t stream) {
  if (!tb.n_tiles) return cudaSuccess;
  venc_emit_kernel<<<tb.n_tiles, kVarThreads, 0, stream>>>(tb);
  return cudaGetLastError();
}
cudaError_t launch_vdec_count(const VarTables& tb, cudaStream_t stream) {
  if (!tb.n_tiles) return cudaSuccess;
  const uint32_t per = kVarThreads / 32;   // one warp per tile
  vdec_count_kernel<<<(tb.n_tiles + per - 1) / per, kVarThreads, 0, stream>>>(tb);
  return cudaGetLastError();
}
cudaError_t launch_vdec_emit(const VarTables& tb, cudaStream_t stream) {
  if (!tb.n_tiles) return cudaSuccess;
  vdec_emit_kernel<<<tb.n_tiles, kVarThreads, 0, stream>>>(tb);
  return cudaGetLastError();
}
cudaError_t launch_vdec_plan(const VarPlan& vp, cudaStream_t stream) {
  vdec_plan_kernel<<<1, kVarPlanThreads, 0, stream>>>(vp);
  return cudaGetLastError();
}
cudaError_t launch_vdec_dev(const VarTables& tb, uint32_t max_ctas, cudaStream_t stream, const VarPadMap* pm) {
  const uint32_t per = kVarThreads / 32;
  vdec_count_dev_kernel<<<std::max(1u, std::min((tb.n_tiles + per - 1) / per, max_ctas)), kVarThreads, 0, stream>>>(tb);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  const uint32_t grid = std::max(1u, std::min(tb.n_tiles, max_ctas));
  if (pm) vdec_emit_padded_kernel<<<grid, kVarThreads, 0, stream>>>(tb, *pm);
  else vdec_emit_dev_kernel<<<grid, kVarThreads, 0, stream>>>(tb);
  return cudaGetLastError();
}

cudaError_t launch_padded(const PaddedPlan& pp, uint32_t emit_grid, cudaStream_t stream, bool strings) {
  if (strings) padded_plan_strings_kernel<<<1, kConcatPlanThreads, 0, stream>>>(pp);
  else padded_plan_kernel<<<1, kConcatPlanThreads, 0, stream>>>(pp);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  padded_emit_kernel<<<std::max(1u, emit_grid), kPadEmitThreads, 0, stream>>>(pp);
  return cudaGetLastError();
}

}  // namespace b200tfs
