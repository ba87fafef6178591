// strcol.h - what the routes over offset-indexed byte columns (Arrow / cuDF layout, b200tfs_bytes) share: the tf.Example encode
// (BytesList.value, tag 0A), the padded encode (TensorProto.string_val, tag 42) and the concatenated decode.
#pragma once
#include "wire.h"

namespace b200tfs {

// Strings at most this long are copied by their own lane, longer ones by the warp (not tuned: DESIGN.md §4.4).
constexpr uint64_t kStrLaneCopy = 64;

// wire bytes of one length-delimited value of `len` bytes: the caller's tag, vi(len), the bytes
B2_HD uint64_t string_value_len(uint64_t len) { return 1 + varint_len(len) + len; }

#if defined(__CUDACC__)
// bytes [0, m) of src to dst by `n` threads (this one is `i`), 16 bytes per thread and step, all 16 loaded before the first
// store.  They wait packed in four words: sixteen byte registers make ex_emit_kernel<kExColumns> spill.
__device__ __forceinline__ void copy_bytes(uint8_t* dst, const uint8_t* src, uint64_t m, uint32_t i, uint32_t n) {
#pragma unroll 1
  for (uint64_t a = (uint64_t)i * 16; a < m; a += (uint64_t)n * 16) {
    uint32_t v[4] = {0, 0, 0, 0};
#pragma unroll
    for (int k = 0; k < 16; ++k) if (a + k < m) v[k >> 2] |= (uint32_t)__ldg(src + a + k) << (8 * (k & 3));
#pragma unroll
    for (int k = 0; k < 16; ++k) if (a + k < m) dst[a + k] = (uint8_t)(v[k >> 2] >> (8 * (k & 3)));
  }
}

// Warp-collective (all 32 lanes call it): each lane's string of `len` bytes from src to dst.  An active lane copies its own string of
// at most kStrLaneCopy bytes; then the warp copies, one by one, every active longer one of at most warp_max bytes (longer: the caller).
__device__ __forceinline__ void warp_copy_strings(uint8_t* dst, const uint8_t* src, uint64_t len, bool active, uint64_t warp_max) {
  if (active && len <= kStrLaneCopy)
    for (uint64_t k = 0; k < len; ++k) dst[k] = src[k];
  uint32_t longs = __ballot_sync(0xFFFFFFFFu, active && len > kStrLaneCopy && len <= warp_max);
#pragma unroll 1
  while (longs) {
    const int l = __ffs(longs) - 1;
    longs &= longs - 1;
    uint8_t* d = (uint8_t*)__shfl_sync(0xFFFFFFFFu, (unsigned long long)(uintptr_t)dst, l);
    const uint8_t* s = (const uint8_t*)__shfl_sync(0xFFFFFFFFu, (unsigned long long)(uintptr_t)src, l);
    copy_bytes(d, s, __shfl_sync(0xFFFFFFFFu, len, l), threadIdx.x & 31, 32);
  }
}
#endif

}  // namespace b200tfs
