// varint_kernels.cuh - packed-varint encode / decode kernels (included by kernels.cu inside
// namespace b200tfs).  Fields: int_val / int64_val / uint32_val / uint64_val / half_val / bool_val.
//
//   encode:  venc_len_kernel   bytes every tile of 2048 elements will occupy -> tile_val[], and by
//                              atomics the sums over groups of 256 tiles and the job total (which the
//                              host needs for the length prefix: b200tfs_measure)
//            venc_emit_kernel  each CTA derives its own output offset (group sums before its group +
//                              tile values before it inside the group), builds every varint in
//                              REGISTERS (7-bit groups spread with three bit-selects per 4 bytes),
//                              appends whole 32-bit words to a shared-memory image of the output that
//                              has the destination's 16-byte phase, and streams the image out with
//                              128-bit stores
//            Each pass is one tile body over a tile source: venc_len_tile and venc_emit_tile.  The two kernels here run
//            them over contiguous segments (SegSrc), unpad_len_kernel and unpad_emit_kernel over the boxes of a padded
//            tensor (BoxSrc, unpad_kernels.cuh).
//   decode:  vdec_count_kernel terminators (bytes with the top bit clear) per tile: an ALIGNED 8 KB window of
//                              the chunk, one warp per tile, sixteen 128-bit loads in flight per lane
//            vdec_emit_kernel  offset as above; finds the varint starts of the tile with bit tricks,
//                              compacts them, and decodes one element per thread from a funnel-shifted
//                              12-byte window (7-bit groups compressed with masks and shifts)
//
// There is no separate scan kernel: a tile's prefix is one coalesced read of <= 256 + n_tiles/256
// counters.  Single-pass encoders and decoders (ticketed tiles with a decoupled look-back over tile or group
// states, or a wait for every predecessor to publish) were tried, measured slower than count + emit, and removed.
// The counting pass is cheap and leaves the wire in L2 for the decoder.
//
// What the reference does here: tensors.py:22 (`.item()` per element into RepeatedScalarContainer,
// the runtime then writes one varint at a time) and tensors.py:46 (list of Python ints -> np.array).

// (a & m) | (b & ~m) in ONE instruction (left to itself the compiler splits it into two masked operations)
__device__ __forceinline__ uint32_t bitsel(uint32_t m, uint32_t a, uint32_t b) {
  uint32_t d;
  asm("lop3.b32 %0, %1, %2, %3, 0xE4;" : "=r"(d) : "r"(a), "r"(b), "r"(m));
  return d;
}

// bytes of the varint of v: bits = position of the top set bit, len = ceil(bits / 7) without a division or a branch
__device__ __forceinline__ uint32_t vlen64(uint64_t v) {
  const uint32_t nb = 64u - (uint32_t)__clzll((long long)(v | 1ull));
  return ((nb + 6u) * 37u) >> 8;   // (nb + 6) / 7 for nb + 6 <= 70
}

// one element of SZ bytes from GLOBAL memory (read-only path), widened to 64 bits the way the protobuf
// runtime widens it: sign-extended for the signed dtypes
template <uint32_t SZ, bool SG>
__device__ __forceinline__ uint64_t ldg_elem(const uint8_t* p) {
  if (SZ == 1) { const uint8_t t = __ldg(p); return SG ? (uint64_t)(int64_t)(int8_t)t : t; }
  if (SZ == 2) { const uint16_t t = __ldg(reinterpret_cast<const uint16_t*>(p)); return SG ? (uint64_t)(int64_t)(int16_t)t : t; }
  if (SZ == 4) { const uint32_t t = __ldg(reinterpret_cast<const uint32_t*>(p)); return SG ? (uint64_t)(int64_t)(int32_t)t : t; }
  return __ldg(reinterpret_cast<const unsigned long long*>(p));
}
// the same for an element type known at run time
__device__ __forceinline__ uint64_t ldg_elem_rt(const uint8_t* p, uint32_t size, uint32_t is_signed) {
  switch (size * 2 + (is_signed ? 1 : 0)) {
    case 2: return ldg_elem<1, false>(p);
    case 3: return ldg_elem<1, true>(p);
    case 4: return ldg_elem<2, false>(p);
    case 5: return ldg_elem<2, true>(p);
    case 8: return ldg_elem<4, false>(p);
    case 9: return ldg_elem<4, true>(p);
    default: return ldg_elem<8, false>(p);
  }
}

// kVarPerThread elements per thread, striped (element base + i*kVarThreads + tid), ALL loads issued
// before any use; a full tile takes the branch without predicates (one base address, immediate offsets)
template <uint32_t SZ, bool SG>
__device__ __forceinline__ void load_striped_t(const uint8_t* src, uint64_t e0, uint32_t cnt, uint64_t (&v)[kVarPerThread]) {
  const uint8_t* base = src + (e0 + threadIdx.x) * SZ;
  if (cnt == kVarTileElems) {
#pragma unroll
    for (uint32_t i = 0; i < kVarPerThread; ++i) v[i] = ldg_elem<SZ, SG>(base + (uint64_t)i * kVarThreads * SZ);
  } else {
#pragma unroll
    for (uint32_t i = 0; i < kVarPerThread; ++i)
      v[i] = (i * kVarThreads + threadIdx.x < cnt) ? ldg_elem<SZ, SG>(base + (uint64_t)i * kVarThreads * SZ) : 0ull;
  }
}

// segment and job of tile t: from the parameter space when there is one of each, else two table look-ups
__device__ __forceinline__ void fetch_tile(const VarTables& tb, uint32_t t, VarSeg& sg, VarJobDev& jb) {
  if (tb.single) { sg = tb.seg0; jb = tb.job0; }
  else { sg = tb.segs[tb.tile_seg[t]]; jb = tb.jobs[sg.job]; }
}

struct VarShared {            // reduction scratch of one CTA
  uint32_t w32[kVarThreads / 32];
  uint64_t w64[kVarThreads / 32];
};

// this thread's share of the tile's prefix: counters of the groups before the tile's group, and of
// the tiles before it inside the group (kVarGroupTiles == kVarThreads: one counter per thread)
__device__ __forceinline__ uint64_t prefix_share(const VarJobDev& jb, uint32_t t_rel) {
  const uint32_t g = t_rel / kVarGroupTiles;
  uint64_t s = 0;
  for (uint32_t i = threadIdx.x; i < g; i += kVarThreads) s += jb.group_sum[i];
  const uint32_t k = g * kVarGroupTiles + threadIdx.x;
  if (k < t_rel) s += jb.tile_val[k];
  return s;
}

// block-wide exclusive scan of `v` (one value per thread) fused with a block-wide sum of `extra`
__device__ __forceinline__ uint32_t block_scan_sum(uint32_t v, uint32_t* total, uint64_t extra, uint64_t* extra_total, VarShared& sh) {
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  uint32_t inc = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t n = __shfl_up_sync(0xFFFFFFFFu, inc, d);
    if (lane >= d) inc += n;
  }
#pragma unroll
  for (int d = 16; d; d >>= 1) extra += __shfl_xor_sync(0xFFFFFFFFu, extra, d);
  if (lane == 31) sh.w32[wid] = inc;
  if (lane == 0) sh.w64[wid] = extra;
  __syncthreads();
  uint32_t base = 0, tot = 0;
  uint64_t etot = 0;
#pragma unroll
  for (uint32_t w = 0; w < kVarThreads / 32; ++w) {
    const uint32_t x = sh.w32[w];
    if (w < wid) base += x;
    tot += x;
    etot += sh.w64[w];
  }
  __syncthreads();
  *total = tot;
  *extra_total = etot;
  return base + inc - v;
}

// block-wide sum; valid in thread 0 only (one barrier)
__device__ __forceinline__ uint32_t block_sum_t0(uint32_t v, VarShared& sh) {
#pragma unroll
  for (int d = 16; d; d >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, d);
  if ((threadIdx.x & 31) == 0) sh.w32[threadIdx.x >> 5] = v;
  __syncthreads();
  uint32_t tot = 0;
  if (threadIdx.x == 0) {
#pragma unroll
    for (uint32_t w = 0; w < kVarThreads / 32; ++w) tot += sh.w32[w];
  }
  return tot;
}

__device__ __forceinline__ void publish_tile(const VarJobDev& jb, uint32_t t_rel, uint32_t total) {
  jb.tile_val[t_rel] = total;
  atomicAdd(&jb.group_sum[t_rel / kVarGroupTiles], total);
  atomicAdd(jb.total, (unsigned long long)total);
}

// E1: the bytes tile t_rel of job `jb` will occupy, elements [e0, e0 + cnt) of `src`, into the job's counters
template <class Src>
__device__ __forceinline__ void venc_len_tile(VarShared& sh, const VarJobDev& jb, uint32_t t_rel, uint64_t e0, uint32_t cnt, const Src& src) {
  uint64_t v[kVarPerThread];
  src.load_striped(e0, cnt, v);
  uint32_t sum = 0;
#pragma unroll
  for (uint32_t i = 0; i < kVarPerThread; ++i) sum += vlen64(v[i]) & ((i * kVarThreads + threadIdx.x < cnt) ? ~0u : 0u);
  const uint32_t total = block_sum_t0(sum, sh);
  if (threadIdx.x == 0) publish_tile(jb, t_rel, total);
}

// 28 value bits -> four 7-bit groups, one per byte; bit 7 of every byte is left dirty for the caller's
// final select (which merges the continuation bits in the same instruction)
__device__ __forceinline__ uint32_t spread28(uint32_t x) {
  const uint32_t t = bitsel(0xFFFF0000u, x << 2, x);   // bits 14..27 -> 16..29
  return bitsel(0xFF00FF00u, t << 1, t);               // bits 7..13 -> 8..14, 23..29 -> 24..30
}

// E2: emit.  Elements are loaded striped (coalesced) and transposed through shared memory (16-byte chunks
// XOR-swizzled by row, so both sides are conflict-free) so that each thread owns kVarPerThread
// consecutive elements; the staging image reuses the same shared memory.
constexpr uint32_t kVarImageBytes = kVarTileElems * 10 + 48;

// The tile's elements, blocked through shared memory: the thread's striped elements (element i * kVarThreads + tid of the tile in
// v[i], as a source's load_striped loads them) are transposed (16-byte chunks XOR-swizzled by row) so that thread r owns
// elements [8r, 8r+8); `lens` and the return value as a source's load_tile gives them.  One barrier inside.
__device__ __forceinline__ uint32_t venc_block_tile(uint8_t* smem, uint32_t cnt, const uint64_t (&v)[kVarPerThread], uint64_t (&mine)[kVarPerThread],
                                                    uint32_t& lens) {
  const uint32_t r = threadIdx.x;
  uint64_t* vals = reinterpret_cast<uint64_t*>(smem);
  {
#pragma unroll
    for (uint32_t i = 0; i < kVarPerThread; ++i) {
      const uint32_t k = i * kVarThreads + threadIdx.x, r = k >> 3, c = k & 7;
      vals[r * 8 + ((((c >> 1) ^ (r >> 1)) & 3) << 1) + (c & 1)] = v[i];
    }
  }
  __syncthreads();
#pragma unroll
  for (uint32_t j = 0; j < kVarPerThread / 2; ++j) {
    const uint4 q = *reinterpret_cast<const uint4*>(smem + r * 64 + (((j ^ (r >> 1)) & 3) << 4));
    mine[2 * j] = (uint64_t)q.x | ((uint64_t)q.y << 32);
    mine[2 * j + 1] = (uint64_t)q.z | ((uint64_t)q.w << 32);
  }
  lens = 0;
#pragma unroll
  for (uint32_t i = 0; i < kVarPerThread; ++i) lens |= vlen64(mine[i]) << (4 * i);
  // elements past the end of the tensor (last tile only) take no room
  const uint32_t have = min(kVarPerThread, cnt - min(cnt, r * kVarPerThread));
  lens &= __funnelshift_lc(0xFFFFFFFFu, 0u, 4u * have);
  const uint32_t pairs = (lens & 0x0F0F0F0Fu) + ((lens >> 4) & 0x0F0F0F0Fu);
  return (pairs * 0x01010101u) >> 24;
}

// Where the elements of an encode tile come from.  A source gives elements [e0, e0 + cnt) of its job in the two forms the passes
// take them:
//   load_striped  element i * kVarThreads + tid of the tile in v[i], every load issued before any use (venc_len_tile)
//   load_tile     blocked: thread r owns elements [8r, 8r+8) of the tile, `lens` = their varint lengths, one nibble each (elements
//                 past the end of the tensor: 0); returns the thread's byte count.  One barrier inside (venc_emit_tile)
// SegSrc is a contiguous segment; BoxSrc (unpad_kernels.cuh) a box cut out of a padded tensor.
struct SegSrc {
  const uint8_t* src;
  uint32_t elem_size, is_signed;

  __device__ __forceinline__ void load_striped(uint64_t e0, uint32_t cnt, uint64_t (&v)[kVarPerThread]) const {
    switch (elem_size * 2 + (is_signed ? 1 : 0)) {
      case 2: load_striped_t<1, false>(src, e0, cnt, v); break;
      case 3: load_striped_t<1, true>(src, e0, cnt, v); break;
      case 4: load_striped_t<2, false>(src, e0, cnt, v); break;
      case 5: load_striped_t<2, true>(src, e0, cnt, v); break;
      case 8: load_striped_t<4, false>(src, e0, cnt, v); break;
      case 9: load_striped_t<4, true>(src, e0, cnt, v); break;
      default: load_striped_t<8, false>(src, e0, cnt, v); break;
    }
  }

  __device__ __forceinline__ uint32_t load_tile(uint8_t* smem, uint64_t e0, uint32_t cnt, uint64_t (&mine)[kVarPerThread], uint32_t& lens) const {
    const uint32_t r = threadIdx.x;
    // 64-bit elements of a full tile whose first byte is 16-byte aligned: every thread loads its own eight consecutive elements
    // with four 128-bit loads - no shared-memory transpose, no barrier (the four loads of a warp cover 2 KB of consecutive bytes
    // between them; each sector is fetched once and served from L1 to the neighbouring instruction)
    const uint8_t* first = src + e0 * 8;
    if (elem_size == 8 && cnt == kVarTileElems && ((uintptr_t)first & 15) == 0) {
      const uint4* p = reinterpret_cast<const uint4*>(first) + 4 * r;
      uint4 q[kVarPerThread / 2];
#pragma unroll
      for (uint32_t j = 0; j < kVarPerThread / 2; ++j) q[j] = __ldg(p + j);
      uint32_t any_hi = 0;
#pragma unroll
      for (uint32_t j = 0; j < kVarPerThread / 2; ++j) {
        mine[2 * j] = (uint64_t)q[j].x | ((uint64_t)q[j].y << 32);
        mine[2 * j + 1] = (uint64_t)q[j].z | ((uint64_t)q[j].w << 32);
        any_hi |= q[j].y | q[j].w;
      }
      lens = 0;
      if (__all_sync(0xFFFFFFFFu, any_hi == 0u)) {      // the warp's values all fit 32 bits: lengths from the low words alone
#pragma unroll
        for (uint32_t i = 0; i < kVarPerThread; ++i) {
          const uint32_t nb = 32u - (uint32_t)__clz((int)((uint32_t)mine[i] | 1u));
          lens |= (((nb + 6u) * 37u) >> 8) << (4 * i);
        }
      } else {
#pragma unroll
        for (uint32_t i = 0; i < kVarPerThread; ++i) lens |= vlen64(mine[i]) << (4 * i);
      }
      const uint32_t pairs = (lens & 0x0F0F0F0Fu) + ((lens >> 4) & 0x0F0F0F0Fu);
      return (pairs * 0x01010101u) >> 24;
    }
    uint64_t v[kVarPerThread];
    load_striped(e0, cnt, v);
    return venc_block_tile(smem, cnt, v, mine, lens);
  }
};

// build the thread's varints in registers and append them, whole 32-bit words at a time, to the shared-memory image at byte
// offset `off`; two barriers inside (every thread must have read its elements out of `smem` before this is called: the
// block scan between the source's load_tile and here has a barrier)
__device__ __forceinline__ void venc_build_image(uint8_t* smem, const uint64_t (&mine)[kVarPerThread], uint32_t lens, uint32_t off) {
  const uint32_t f0 = off & 3;
  const uint32_t sbase = (uint32_t)__cvta_generic_to_shared(smem);
  const uint32_t sa0 = sbase + (off & ~3u);      // shared-window address of the word being filled
  uint32_t sa = sa0, f = f0, acc = 0;
  // Every varint of the warp fits four bytes (values below 2^28: token ids, indices, class labels, small counts - the bulk of
  // what int_val / int64_val carry in practice)?  Then an element is one spread word, completes at most one 32-bit word of the
  // image, and the upper half of the value is never looked at: ~20 instructions per element instead of ~45.
  const bool narrow = __all_sync(0xFFFFFFFFu, ((lens + 0x33333333u) & 0x88888888u) == 0u);   // every nibble <= 4
  if (narrow) {
#pragma unroll
    for (uint32_t i = 0; i < kVarPerThread; ++i) {
      const uint32_t lo = (uint32_t)mine[i];
      const uint32_t L = (lens >> (4 * i)) & 15u;
      const uint32_t w0 = bitsel(0x7F7F7F7Fu, spread28(lo), __funnelshift_lc(0xFFFFFFFFu, 0u, 8u * L - 8u));   // L = 0: see below
      const uint32_t shb = f * 8u;
      const uint32_t o0 = acc | (w0 << shb);
      const uint32_t o1 = __funnelshift_l(w0, 0u, shb);
      const uint32_t n = f + L;
      asm volatile(
          "{\n\t.reg .pred p0;\n\t"
          "setp.ge.u32 p0, %1, 4;\n\t"
          "@p0 st.shared.u32 [%2], %3;\n\t"
          "selp.b32 %0, %4, %3, p0;\n\t}"
          : "=r"(acc) : "r"(n), "r"(sa), "r"(o0), "r"(o1) : "memory");
      sa += n & ~3u;
      f = n & 3;
    }
  } else {
#pragma unroll
    for (uint32_t i = 0; i < kVarPerThread; ++i) {
      const uint32_t lo = (uint32_t)mine[i], hi = (uint32_t)(mine[i] >> 32);
      const uint32_t L = (lens >> (4 * i)) & 15u;
      // continuation bits go into the first L-1 bytes: the low 8(L-1) bits of a mask, by a clamped funnel shift.  (An
      // absent element - only at the end of the last tile - has L = 0: what it ORs into `acc` lies above byte f and is
      // never stored, because no element follows it.)
      const uint32_t s = 8u * L - 8u;
      const uint32_t w0 = bitsel(0x7F7F7F7Fu, spread28(lo), __funnelshift_lc(0xFFFFFFFFu, 0u, s));
      uint32_t w1 = 0, w2 = 0;
      if (L > 4) {
        w1 = bitsel(0x7F7F7F7Fu, spread28(__funnelshift_r(lo, hi, 28)), __funnelshift_lc(0xFFFFFFFFu, 0u, s - 32u));
        const uint32_t x2 = hi >> 24;          // bits 56..63: byte 8 carries seven of them, byte 9 the last one ...
        w2 = x2 | ((x2 & 0x80u) << 1);         // ... and when that one is set, byte 8 continues: the same bit
      }
      const uint32_t shb = f * 8u;
      const uint32_t o0 = acc | (w0 << shb);
      const uint32_t o1 = __funnelshift_l(w0, w1, shb);
      const uint32_t o2 = __funnelshift_l(w1, w2, shb);
      const uint32_t o3 = __funnelshift_l(w2, 0u, shb);
      const uint32_t n = f + L;
      // store the words this element completed; keep the incomplete one
      asm volatile(
          "{\n\t.reg .pred p0, p1, p2;\n\t.reg .b32 t;\n\t"
          "setp.ge.u32 p0, %1, 4;\n\tsetp.ge.u32 p1, %1, 8;\n\tsetp.ge.u32 p2, %1, 12;\n\t"
          "@p0 st.shared.u32 [%2], %3;\n\t@p1 st.shared.u32 [%2+4], %4;\n\t@p2 st.shared.u32 [%2+8], %5;\n\t"
          "selp.b32 t, %4, %3, p0;\n\tselp.b32 t, %5, t, p1;\n\tselp.b32 %0, %6, t, p2;\n\t}"
          : "=r"(acc) : "r"(n), "r"(sa), "r"(o0), "r"(o1), "r"(o2), "r"(o3) : "memory");
      sa += n & ~3u;
      f = n & 3;
    }
  }
  __syncthreads();
  // the word this thread did not complete: its bytes only (the thread that completes the word stored zeros there)
  {
    const uint32_t first = (sa == sa0) ? f0 : 0u;
    uint8_t* tail = smem + (sa - sbase);
#pragma unroll
    for (uint32_t b = 0; b < 3; ++b)
      if (b >= first && b < f) tail[b] = (uint8_t)(acc >> (8 * b));
  }
  __syncthreads();
}

// E2: tile t_rel of job `jb`, elements [e0, e0 + cnt) of `src`.  The offset comes from the counters, src.load_tile fills the
// registers, then the image and the stores.
template <class Src>
__device__ __forceinline__ void venc_emit_tile(uint8_t* smem, VarShared& sh, const VarJobDev& jb, uint32_t t_rel, uint64_t e0, uint32_t cnt,
                                               const Src& src) {
  const uint64_t share = prefix_share(jb, t_rel);
  uint64_t mine[kVarPerThread];
  uint32_t lens;
  const uint32_t sum = src.load_tile(smem, e0, cnt, mine, lens);
  uint32_t total;
  uint64_t base;
  uint32_t off = block_scan_sum(sum, &total, share, &base, sh);   // every thread has read its elements before the first barrier inside
  uint8_t* g = jb.dst + base;                  // first output byte of this tile
  const uint32_t phase = (uint32_t)((uintptr_t)g & 15);
  venc_build_image(smem, mine, lens, off + phase);
  // smem[phase .. phase+total) -> g[0 .. total); whole 16-byte vectors where the tile owns them.  Never past the
  // payload the header announced (the data changed between b200tfs_measure and the encode: undefined bytes, no overrun)
  if (base >= jb.cap) return;
  total = (uint32_t)min((uint64_t)total, jb.cap - base);
  uint8_t* gbase = g - phase;  // 16-byte aligned
  const uint32_t lo = phase, hi = phase + total;
  const uint32_t v_lo = (lo + 15) >> 4, v_hi = hi >> 4;
  if (v_lo < v_hi) {
    // stepped by byte offset: stepped by vector index, the unrolled loop kept two more induction variables, and venc_emit_kernel spilled more
    for (uint32_t o = 16 * (v_lo + threadIdx.x); o < 16 * v_hi; o += 16 * kVarThreads) st_stream(gbase + o, *reinterpret_cast<const uint4*>(smem + o));
    for (uint32_t i = lo + threadIdx.x; i < v_lo * 16; i += kVarThreads) gbase[i] = smem[i];
    for (uint32_t i = v_hi * 16 + threadIdx.x; i < hi; i += kVarThreads) gbase[i] = smem[i];
  } else {
    for (uint32_t i = lo + threadIdx.x; i < hi; i += kVarThreads) gbase[i] = smem[i];
  }
}

__global__ void __launch_bounds__(kVarThreads) venc_len_kernel(const __grid_constant__ VarTables tb) {
  __shared__ VarShared sh;
  const uint32_t t = blockIdx.x;
  VarSeg sg;
  VarJobDev jb;
  fetch_tile(tb, t, sg, jb);
  const uint64_t e0 = (uint64_t)(t - sg.first_tile) * kVarTileElems;
  venc_len_tile(sh, jb, t - jb.first_tile, e0, (uint32_t)min((uint64_t)kVarTileElems, sg.n - e0), SegSrc{sg.src, jb.elem_size, jb.is_signed});
}

__global__ void __launch_bounds__(kVarThreads, 5) venc_emit_kernel(const __grid_constant__ VarTables tb) {
  __shared__ __align__(16) uint8_t smem[kVarImageBytes];
  __shared__ VarShared sh;
  const uint32_t t = blockIdx.x;
  VarSeg sg;
  VarJobDev jb;
  fetch_tile(tb, t, sg, jb);
  const uint64_t e0 = (uint64_t)(t - sg.first_tile) * kVarTileElems;
  venc_emit_tile(smem, sh, jb, t - jb.first_tile, e0, (uint32_t)min((uint64_t)kVarTileElems, sg.n - e0), SegSrc{sg.src, jb.elem_size, jb.is_signed});
}

// D1: varint terminators (bytes with the top bit clear) per decode tile.  One WARP per tile: sixteen
// aligned 128-bit loads per lane in two batches of eight, a warp reduction, no block barrier.
__device__ __forceinline__ void vdec_count_tile(const VarTables& tb, uint32_t t, uint32_t lane) {
  VarSeg sg;
  VarJobDev jb;
  fetch_tile(tb, t, sg, jb);
  const uint8_t* lo = sg.src;
  const uint8_t* hi = sg.src + sg.n;
  const uint8_t* G = reinterpret_cast<const uint8_t*>((uintptr_t)sg.src & ~(uintptr_t)15) + (uint64_t)(t - sg.first_tile) * kVarTileBytes;
  uint32_t cnt = 0;
  constexpr uint32_t kBlocks = kVarTileBytes / 16, kBatch = 8;
  if (G >= lo && G + kVarTileBytes <= hi) {       // interior tile: no edge handling at all
#pragma unroll
    for (uint32_t b = 0; b < kBlocks / 32; b += kBatch) {
      uint4 v[kBatch];
#pragma unroll
      for (uint32_t i = 0; i < kBatch; ++i) v[i] = ld_reuse(G + 16 * (lane + 32 * (b + i)));
#pragma unroll
      for (uint32_t i = 0; i < kBatch; ++i)
        cnt += __popc(~v[i].x & 0x80808080u) + __popc(~v[i].y & 0x80808080u) + __popc(~v[i].z & 0x80808080u) + __popc(~v[i].w & 0x80808080u);
    }
  } else {
    for (uint32_t k = lane; k < kBlocks; k += 32) {
      const uint8_t* p = G + 16 * k;
      if (p >= lo && p + 16 <= hi) {
        const uint4 v = ld_reuse(p);
        cnt += __popc(~v.x & 0x80808080u) + __popc(~v.y & 0x80808080u) + __popc(~v.z & 0x80808080u) + __popc(~v.w & 0x80808080u);
      } else if (p + 16 > lo && p < hi) {
        for (int i = 0; i < 16; ++i) if (p + i >= lo && p + i < hi) cnt += !(p[i] & 0x80);
      }
    }
  }
#pragma unroll
  for (int d = 16; d; d >>= 1) cnt += __shfl_xor_sync(0xFFFFFFFFu, cnt, d);
  if (lane == 0) publish_tile(jb, t - jb.first_tile, cnt);
}
__global__ void __launch_bounds__(kVarThreads, 5) vdec_count_kernel(const __grid_constant__ VarTables tb) {
  const uint32_t t = blockIdx.x * (kVarThreads / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (t >= tb.n_tiles) return;
  vdec_count_tile(tb, t, lane);
}
// the same over tables vdec_plan_kernel built: the tile count is in device memory, the grid a fixed bound (warp-stride loop)
__global__ void __launch_bounds__(kVarThreads, 5) vdec_count_dev_kernel(const __grid_constant__ VarTables tb) {
  const uint32_t nt = *tb.n_tiles_dev, lane = threadIdx.x & 31;
  for (uint32_t t = blockIdx.x * (kVarThreads / 32) + (threadIdx.x >> 5); t < nt; t += gridDim.x * (kVarThreads / 32)) vdec_count_tile(tb, t, lane);
}

// An output's status in the reference's order: FromString refuses a malformed varint (E_PARSE) before np.array() refuses an
// out-of-range value (E_RANGE), which comes before reshape() refuses the element count (E_SHAPE).  The numeric codes do not
// sort that way (E_RANGE < E_PARSE < E_SHAPE), so the status word is raised by rank, not by atomicMin.  Any other code
// (E_NONCANONICAL from the plan) outranks all three: the job never ran.
__device__ __forceinline__ uint32_t var_status_rank(int32_t s) {
  return s == B200TFS_OK ? 0u : s == B200TFS_E_SHAPE ? 1u : s == B200TFS_E_RANGE ? 2u : s == B200TFS_E_PARSE ? 3u : 4u;
}
__device__ __forceinline__ void var_status_raise(int32_t* status, int32_t s) {
  int32_t cur = *reinterpret_cast<volatile int32_t*>(status);
  while (var_status_rank(s) > var_status_rank(cur)) {
    const int32_t seen = atomicCAS(status, cur, s);
    if (seen == cur) break;
    cur = seen;
  }
}

// how a decoded value is stored
enum VarStore : int { VS_U64, VS_U32, VS_I16, VS_I8, VS_U16, VS_U8, VS_BOOL, VS_HALF_BITS, VS_HALF_VALUE };
// does the value fit the element type (int_val carries the 16- and 8-bit types as 32-bit ints: np.array() checks the range)
template <int K>
__device__ __forceinline__ bool decoded_in_range(uint64_t v) {
  const int32_t x = (int32_t)(uint32_t)v;
  if (K == VS_I16) return x >= -32768 && x <= 32767;
  if (K == VS_I8) return x >= -128 && x <= 127;
  if (K == VS_U16) return x >= 0 && x <= 65535;
  if (K == VS_U8) return x >= 0 && x <= 255;
  return true;
}
template <int K>
__device__ __forceinline__ void store_decoded(uint8_t* d, uint64_t idx, uint64_t v) {
  const int32_t x = (int32_t)(uint32_t)v;
  if (K == VS_U64) reinterpret_cast<uint64_t*>(d)[idx] = v;
  else if (K == VS_U32) reinterpret_cast<uint32_t*>(d)[idx] = (uint32_t)v;
  else if (K == VS_I16) reinterpret_cast<int16_t*>(d)[idx] = (int16_t)x;
  else if (K == VS_I8) reinterpret_cast<int8_t*>(d)[idx] = (int8_t)x;
  else if (K == VS_U16) reinterpret_cast<uint16_t*>(d)[idx] = (uint16_t)x;
  else if (K == VS_U8) d[idx] = (uint8_t)x;
  else if (K == VS_BOOL) d[idx] = v != 0;
  else if (K == VS_HALF_BITS) reinterpret_cast<uint16_t*>(d)[idx] = (uint16_t)v;
  else reinterpret_cast<uint16_t*>(d)[idx] = __half_as_ushort(__int2half_rn(x));
}

// four bytes of 7-bit groups -> 28 contiguous bits (continuation bits dropped)
__device__ __forceinline__ uint32_t compress28(uint32_t y) {
  y &= 0x7F7F7F7Fu;
  y = (y & 0x007F007Fu) | ((y & 0x7F007F00u) >> 1);
  return (y & 0x00003FFFu) | ((y >> 2) & 0x0FFFC000u);
}

// bytes up to and including the first terminator of `t` (terminator flags at bit 7 of each byte) kept, the rest cleared
__device__ __forceinline__ uint32_t through_terminator(uint32_t t) { return ((t & (0u - t)) << 1) - 1u; }

// the padded position (in elements from the record's first row) of element e of job `job` (VarPadMap)
__device__ __forceinline__ uint64_t var_pad_index(const VarPadMap& pm, uint32_t job, uint64_t e) {
  const uint32_t r = job / kFusedMaxOutputs, k = job % kFusedMaxOutputs;
  const PadDesc& d = pm.desc[(size_t)r * pm.n_keys + k];
  const PadKeyDev& key = pm.keys[k];
  uint64_t own_row = 1, dst_row = 1;
  for (int32_t a = 1; a < key.rank; ++a) { own_row *= (uint64_t)d.dims[a]; dst_row *= (uint64_t)key.dims[a]; }
  const uint64_t lr = e / own_row;
  uint64_t x = e - lr * own_row, at = 0, stride = 1;
  for (int32_t a = key.rank - 1; a >= 1; --a) {
    const uint64_t q = x / (uint64_t)d.dims[a];
    at += (x - q * (uint64_t)d.dims[a]) * stride;
    stride *= (uint64_t)key.dims[a];
    x = q;
  }
  return lr * dst_row + at;
}

// element j of the tile starts at smraw[start_at[j]]: 12-byte window by funnel shifts, cut after its terminator.
// Two shapes, chosen per warp: every lane's varint ends inside its first four bytes (values below 2^28:
// indices, token ids, small counts), or the general branch-free form.  A varint that never terminates inside the
// chunk is caught by the caller (the chunk's last byte has its continuation bit set); here only the eleven-byte case.
// PAD: element idx0 + j goes to its padded position (var_pad_index) instead of the next one in flat order.
template <int K, bool PAD = false>
__device__ __forceinline__ int32_t decode_elems(const uint8_t* smraw, const uint16_t* start_at, uint32_t n_here,
                                                uint8_t* dst, uint64_t idx0, uint64_t n_elems, const VarPadMap& pm = VarPadMap{},
                                                uint32_t job = 0) {
  int32_t st = B200TFS_OK;
  const uint64_t room = n_elems > idx0 ? n_elems - idx0 : 0;   // elements of the tensor this tile may still write
  const uint32_t n_store = (uint32_t)min((uint64_t)n_here, room);
  uint8_t* out = dst + idx0 * (K == VS_U64 ? 8 : K == VS_U32 ? 4 : (K == VS_I8 || K == VS_U8 || K == VS_BOOL) ? 1 : 2);
  for (uint32_t j0 = 0; j0 < n_here; j0 += kVarThreads) {      // trip count uniform across the CTA
    const uint32_t j = j0 + threadIdx.x;
    const uint32_t q = (j < n_here) ? start_at[j] : 16u;
    const uint32_t* wp = reinterpret_cast<const uint32_t*>(smraw + (q & ~3u));
    const uint32_t shb = (q & 3u) * 8u;
    const uint32_t a0 = wp[0], a1 = wp[1];
    const uint32_t b0 = __funnelshift_r(a0, a1, shb);
    const uint32_t t0 = ~b0 & 0x80808080u;
    uint32_t v_lo, v_hi = 0;
    if (__all_sync(0xFFFFFFFFu, t0 != 0u)) {
      v_lo = compress28(b0 & through_terminator(t0));
    } else {
      const uint32_t a2 = wp[2], a3 = wp[3];
      const uint32_t b1 = __funnelshift_r(a1, a2, shb), b2 = __funnelshift_r(a2, a3, shb);
      const uint32_t t1 = ~b1 & 0x80808080u, t2 = ~b2 & 0x00008080u;
      const uint32_t m0 = t0 ? through_terminator(t0) : 0xFFFFFFFFu;
      const uint32_t m1 = t0 ? 0u : (t1 ? through_terminator(t1) : 0xFFFFFFFFu);
      const uint32_t m2 = (t0 | t1) ? 0u : through_terminator(t2);
      if ((t0 | t1 | t2) == 0u && j < n_here) st = B200TFS_E_PARSE;       // more than ten bytes
      const uint32_t c0 = compress28(b0 & m0), c1 = compress28(b1 & m1), c2 = compress28(b2 & m2);
      v_lo = c0 | (c1 << 28);
      v_hi = (c1 >> 4) | (c2 << 24);
    }
    const uint64_t v = (uint64_t)v_lo | ((uint64_t)v_hi << 32);
    // every value is range-checked, stored or not (a wrong element count stores nothing, yet np.array() sees every value)
    if (j < n_here && !decoded_in_range<K>(v) && st != B200TFS_E_PARSE) st = B200TFS_E_RANGE;
    if (j < n_store) {
      if (PAD) store_decoded<K>(dst, var_pad_index(pm, job, idx0 + j), v);
      else store_decoded<K>(out, j, v);
    }
  }
  return st;
}

// D2: decode.  The tile (an aligned window of the chunk) is staged in shared memory between one 16-byte block of
// look-behind and one of look-ahead, bytes outside the chunk zeroed; each thread owns two 16-byte blocks and
// finds the varints that START there (previous byte is a terminator - the zero before the chunk's first byte
// is one); a block scan ranks them; they are compacted into a list so that the decode step hands out
// ELEMENTS, not byte blocks, to threads: balanced work and coalesced stores.
template <bool PAD = false>
__device__ __forceinline__ void vdec_emit_tile(const VarTables& tb, uint32_t t, const VarPadMap& pm = VarPadMap{}) {
  constexpr uint32_t kBlocks = kVarTileBytes / 16;             // 512: two per thread
  __shared__ __align__(16) uint8_t smraw[16 + kVarTileBytes + 16];
  __shared__ uint16_t start_at[kVarTileBytes];
  __shared__ VarShared sh;
  VarSeg sg;
  VarJobDev jb;
  fetch_tile(tb, t, sg, jb);
  // element count != prod(shape): reshape() would raise.  The tile still looks for malformed varints and out-of-range values
  // (nothing is stored): both are refused before any reshape (var_status_raise)
  const bool count_ok = (jb.flags & kVarFlagPadEdge) ? *jb.total <= jb.n_elems : *jb.total == jb.n_elems;
  if (!count_ok && threadIdx.x == 0) var_status_raise(jb.status, B200TFS_E_SHAPE);
  const uint64_t n_store = count_ok ? jb.n_elems : 0;
  const uint64_t share = prefix_share(jb, t - jb.first_tile);
  const uint8_t* lo = sg.src;
  const uint8_t* hi = sg.src + sg.n;
  const uint8_t* G = reinterpret_cast<const uint8_t*>((uintptr_t)sg.src & ~(uintptr_t)15) + (uint64_t)(t - sg.first_tile) * kVarTileBytes;
  // stage blocks -1 .. kBlocks (smraw[16 * (k + 1)] <- G[16 * k]); whole blocks inside the chunk move as vectors
  auto stage = [&](int32_t k) {
    const uint8_t* p = G + 16 * (int64_t)k;
    uint8_t* s = smraw + 16 * (k + 1);
    if (p >= lo && p + 16 <= hi) *reinterpret_cast<uint4*>(s) = ld_stream(p);
    else {
      uint4 z = make_uint4(0u, 0u, 0u, 0u);
      *reinterpret_cast<uint4*>(s) = z;
      if (p + 16 > lo && p < hi)
        for (int i = 0; i < 16; ++i) if (p + i >= lo && p + i < hi) s[i] = p[i];
    }
  };
  stage((int32_t)threadIdx.x);
  stage((int32_t)(threadIdx.x + kVarThreads));
  if (threadIdx.x < 2) stage(threadIdx.x == 0 ? -1 : (int32_t)kBlocks);
  __syncthreads();
  // Phase 1 - find the starts: one conflict-free 128-bit shared load per block, then bit tricks.  A varint
  // STARTS at byte i when byte i-1 has its top bit clear.
  uint32_t startm[2];
#pragma unroll
  for (uint32_t r = 0; r < 2; ++r) {
    const uint32_t k = threadIdx.x + r * kVarThreads;
    const uint8_t* s = smraw + 16 * (k + 1);
    const uint4 w = *reinterpret_cast<const uint4*>(s);
    auto msb4 = [](uint32_t x) { return (((x >> 7) & 0x01010101u) * 0x01020408u) >> 24; };   // 4 top bits -> nibble
    const uint32_t cont = msb4(w.x) | (msb4(w.y) << 4) | (msb4(w.z) << 8) | (msb4(w.w) << 12);
    const uint32_t prev_term = (s[-1] & 0x80) ? 0u : 1u;
    uint32_t st = (((~cont) << 1) | prev_term) & 0xFFFFu;
    const uint8_t* p = G + 16 * k;
    if (!(p >= lo && p + 16 <= hi)) {              // block straddles an end of the chunk: positions inside it only
      const int64_t first = max((int64_t)0, min((int64_t)16, (int64_t)(lo - p))), last = max((int64_t)0, min((int64_t)16, (int64_t)(hi - p)));
      st &= ((1u << last) - 1u) & ~((1u << first) - 1u);
    }
    startm[r] = st;
  }
  // Phase 2 - rank them in position order (second-round blocks lie after every first-round block): one scan
  // over both counts packed into a word, fused with the reduction that yields the tile's element offset
  const uint32_t packed = __popc(startm[0]) | (__popc(startm[1]) << 16);
  uint32_t packed_total;
  uint64_t before;
  const uint32_t rank = block_scan_sum(packed, &packed_total, share, &before, sh);
  const uint32_t first_total = packed_total & 0xFFFFu, n_here = first_total + (packed_total >> 16);
#pragma unroll
  for (uint32_t r = 0; r < 2; ++r) {
    uint32_t starts = startm[r], at = (r == 0) ? (rank & 0xFFFFu) : first_total + (rank >> 16);
    const uint32_t at0 = 16 * (threadIdx.x + r * kVarThreads + 1);
    while (starts) {
      const uint32_t i = __ffs(starts) - 1;
      starts &= starts - 1;
      start_at[at++] = (uint16_t)(at0 + i);
    }
  }
  __syncthreads();
  // Phase 3 - the index of an element in the tensor is the number of terminators before it: `before`
  // counts those ahead of the tile (+1 when a varint straddles in from the previous tile: it precedes ours but
  // its terminator is here).
  const uint64_t idx0 = before + (smraw[15] >> 7);
  if (threadIdx.x == 0 && hi > G && hi <= G + kVarTileBytes && (hi[-1] & 0x80)) var_status_raise(jb.status, B200TFS_E_PARSE);   // the chunk's last varint never ends
  int32_t st_local;
  const uint32_t job = sg.job;
  switch (jb.dtype) {
    case DT_INT64: case DT_UINT64: st_local = decode_elems<VS_U64, PAD>(smraw, start_at, n_here, jb.dst, idx0, n_store, pm, job); break;
    case DT_INT32: case DT_UINT32: st_local = decode_elems<VS_U32, PAD>(smraw, start_at, n_here, jb.dst, idx0, n_store, pm, job); break;
    case DT_INT16: st_local = decode_elems<VS_I16, PAD>(smraw, start_at, n_here, jb.dst, idx0, n_store, pm, job); break;
    case DT_INT8: st_local = decode_elems<VS_I8, PAD>(smraw, start_at, n_here, jb.dst, idx0, n_store, pm, job); break;
    case DT_UINT16: st_local = decode_elems<VS_U16, PAD>(smraw, start_at, n_here, jb.dst, idx0, n_store, pm, job); break;
    case DT_UINT8: st_local = decode_elems<VS_U8, PAD>(smraw, start_at, n_here, jb.dst, idx0, n_store, pm, job); break;
    case DT_BOOL: st_local = decode_elems<VS_BOOL, PAD>(smraw, start_at, n_here, jb.dst, idx0, n_store, pm, job); break;
    case DT_HALF: case DT_BFLOAT16:
      st_local = (jb.flags & kVarFlagHalfAsValue) ? decode_elems<VS_HALF_VALUE, PAD>(smraw, start_at, n_here, jb.dst, idx0, n_store, pm, job)
                                                  : decode_elems<VS_HALF_BITS, PAD>(smraw, start_at, n_here, jb.dst, idx0, n_store, pm, job);
      break;
    default: st_local = B200TFS_OK; break;
  }
  if (st_local != B200TFS_OK) var_status_raise(jb.status, st_local);
}
__global__ void __launch_bounds__(kVarThreads) vdec_emit_kernel(const __grid_constant__ VarTables tb) { vdec_emit_tile(tb, blockIdx.x); }
// the same over tables vdec_plan_kernel built (grid-stride loop; the barrier keeps the next tile's staging behind this one's reads)
__global__ void __launch_bounds__(kVarThreads) vdec_emit_dev_kernel(const __grid_constant__ VarTables tb) {
  const uint32_t nt = *tb.n_tiles_dev;
  for (uint32_t t = blockIdx.x; t < nt; t += gridDim.x) {
    vdec_emit_tile(tb, t);
    __syncthreads();
  }
}
// the same for the padded decode (b200tfs_decode_padded): every element goes to its padded position
__global__ void __launch_bounds__(kVarThreads) vdec_emit_padded_kernel(const __grid_constant__ VarTables tb, const __grid_constant__ VarPadMap pm) {
  const uint32_t nt = *tb.n_tiles_dev;
  for (uint32_t t = blockIdx.x; t < nt; t += gridDim.x) {
    vdec_emit_tile<true>(tb, t, pm);
    __syncthreads();
  }
}

// Plan of the packed-varint outputs of a single-launch decode (b200tfs_set_decode_varints), on the device: one CTA reads the
// table the fused launch just published, gives output k of record r the fixed job r * kFusedMaxOutputs + k and its runs the
// fixed segments behind it, scans the tile counts (one block scan per kVarPlanThreads slots, the carry in a register), writes
// the tile -> segment map, zeroes the counters and leaves the tile count for the count / emit kernels.  Nothing waits on
// another CTA; a captured graph replays it as it is.
__global__ void __launch_bounds__(kVarPlanThreads) vdec_plan_kernel(const __grid_constant__ VarPlan vp) {
  __shared__ unsigned long long warp_sum[kVarPlanThreads / 32];
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const uint32_t slots = vp.n * (uint32_t)kFusedMaxOutputs;
  unsigned long long carry = 0;     // tiles (low 32 bits) and counter groups (high 32 bits) of the slots before this round
  for (uint32_t s0 = 0; s0 < slots; s0 += kVarPlanThreads) {
    const uint32_t s = s0 + threadIdx.x, r = s / kFusedMaxOutputs, k = s % kFusedMaxOutputs;
    int32_t st = kVarSlotIdle;
    uint32_t tiles = 0, n_runs = 0;
    const b200tfs_output* o = vp.outs + s;
    const uint8_t* rec = nullptr;
    if (s < slots && vp.rec_status[r] == B200TFS_OK && (int32_t)k < vp.n_outs[r] && o->status == B200TFS_OK && o->n_elems &&
        (dtype_info(o->dtype).kind == VK_VARINT || dtype_info(o->dtype).kind == VK_BOOL)) {
      rec = vp.w + (vp.n <= (uint32_t)kFusedInlineRecs ? vp.off_inl[r] : vp.rec_off[r]);
      n_runs = (uint32_t)o->n_runs;
      st = B200TFS_OK;
      // rows of unpacked elements (and more runs than the table holds) are left to b200tfs_unpack_outputs, which gathers them
      if ((o->flags & (B200TFS_OF_UNPACKED | B200TFS_OF_SPILLED)) || o->n_inline != n_runs || n_runs > B200TFS_MAX_RUNS) st = B200TFS_E_NONCANONICAL;
      for (uint32_t q = 0; q < n_runs && st == B200TFS_OK; ++q) {
        if (o->runs[q].count != 1) st = B200TFS_E_NONCANONICAL;
        else tiles += (uint32_t)var_decode_tiles(rec + o->runs[q].off, o->runs[q].len);
      }
      if (st != B200TFS_OK) { tiles = 0; n_runs = 0; }
    }
    const uint32_t groups = (tiles + kVarGroupTiles - 1) / kVarGroupTiles;
    // block-wide exclusive scan of (tiles, groups) packed in 64 bits
    const unsigned long long v = (unsigned long long)tiles | ((unsigned long long)groups << 32);
    unsigned long long inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const unsigned long long x = __shfl_up_sync(0xFFFFFFFFu, inc, d);
      if (lane >= (uint32_t)d) inc += x;
    }
    if (lane == 31) warp_sum[wid] = inc;
    __syncthreads();
    unsigned long long before = carry, round = 0;
    for (uint32_t w = 0; w < kVarPlanThreads / 32; ++w) {
      const unsigned long long x = warp_sum[w];
      if (w < wid) before += x;
      round += x;
    }
    __syncthreads();
    before += inc - v;
    carry += round;
    const uint32_t first_tile = (uint32_t)before, first_group = (uint32_t)(before >> 32);
    // beyond the host's bound (never: var_record_tile_bound) - the tiles inside it still run, but can never match the count
    const bool over = st == B200TFS_OK && first_tile + tiles > vp.tile_cap;
    if (s < slots) {
      vp.status[s] = over ? B200TFS_E_NONCANONICAL : st;
      vp.total[s] = 0;
      VarJobDev jb{};
      if (st == B200TFS_OK) {
        jb.dst = vp.dst + (uint64_t)r * vp.dst_stride + o->dst_off;
        jb.n_elems = over ? ~0ull : o->n_elems;
        jb.dtype = o->dtype;
        jb.elem_size = dtype_info(o->dtype).elem_size;
        jb.is_signed = dtype_info(o->dtype).is_signed;
        jb.first_tile = first_tile;
        jb.n_tiles = tiles;
        jb.tile_val = vp.tile_val + first_tile;
        jb.group_sum = vp.group_sum + first_group;
        jb.total = vp.total + s;
        jb.status = vp.status + s;
        const uint32_t run_tiles = over ? vp.tile_cap - min(first_tile, vp.tile_cap) : tiles;   // the tiles that will run
        for (uint32_t g = 0; g < (run_tiles + kVarGroupTiles - 1) / kVarGroupTiles; ++g) jb.group_sum[g] = 0;
        uint32_t t = first_tile;
        for (uint32_t q = 0; q < n_runs; ++q) {
          const uint8_t* src = rec + o->runs[q].off;
          const uint32_t len = o->runs[q].len, nt = (uint32_t)var_decode_tiles(src, len);
          const uint32_t seg = s * B200TFS_MAX_RUNS + q;
          vp.segs[seg] = VarSeg{src, len, s, t};
          for (uint32_t i = 0; i < nt && t + i < vp.tile_cap; ++i) vp.tile_seg[t + i] = seg;
          t += nt;
        }
      }
      vp.jobs[s] = jb;
    }
  }
  if (threadIdx.x == 0) *vp.n_tiles = (uint32_t)min((unsigned long long)vp.tile_cap, carry & 0xFFFFFFFFull);
}
