// store_path_probe.cu - which store path reaches HBM fastest on sm_90a (NOT part of the product).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o build/store_path_probe tools/store_path_probe.cu
// Run:   build/store_path_probe [runs=3] [launches=20]
//
// Every variant moves 1 GiB per launch (far more than the 50 MB L2), shaped like the kernels of the C2 step: 256 threads, 32 KB
// per round, 64 KB tiles for the encode-shaped (register) variants and 256 KB tiles for the decode-shaped (TMA-in) ones.  Each
// variant is timed with CUDA events over `launches` launches after three warm-up launches; the variants alternate within each
// of `runs` runs.  GB/s counts read + write bytes.  The CTAs resident per SM are pinned with dynamic shared memory padding and
// printed as the occupancy API reports them.
//   write-only : cudaMemsetAsync | st.global.L1::no_allocate.v4 from registers | TMA bulk store (cp.async.bulk.global.shared::cta)
//   read-only  : ld.global.nc.L1::no_allocate.v4 + reduction | TMA bulk loads into shared memory
//   1:1 copy   : reg in -> st.global out (move_kernel's body_aligned) | TMA in -> st.global out (the staged decode)
//                | TMA in -> smem -> TMA out | reg in -> smem -> TMA out; each at 1, 2, 3 CTAs/SM, the TMA / st.global stores
//                also with an L2 evict-first policy (createpolicy)
//   1:2 widen  : body_widen (reg in, two st.global out per unit) | TMA in, widen into shared memory, TMA out
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <algorithm>
#include <functional>
#include <string>
#include <vector>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); exit(1); } } while (0)

constexpr uint32_t kT = 256;            // threads per CTA (kMoveThreads)
constexpr uint32_t kRoundBytes = 32768; // 8 x 16 B per thread

// ---- global accessors (as kernels.cu) ----
__device__ __forceinline__ uint4 ld_stream(const uint8_t* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ void st_stream(uint8_t* p, const uint4& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" :: "l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ void st_stream_hint(uint8_t* p, const uint4& v, uint64_t pol) {
  asm volatile("st.global.L1::no_allocate.L2::cache_hint.v4.u32 [%0], {%1,%2,%3,%4}, %5;"
               :: "l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w), "l"(pol) : "memory");
}
__device__ __forceinline__ uint64_t evict_first_policy() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ uint32_t quiet(uint32_t w) { return ((w & 0x7FFFFFFFu) > 0x7F800000u) ? (w | 0x00400000u) : w; }
__device__ __forceinline__ uint4 fix(uint4 v) { v.x = quiet(v.x); v.y = quiet(v.y); v.z = quiet(v.z); v.w = quiet(v.w); return v; }
__device__ __forceinline__ uint32_t widen(uint32_t h) { return __float_as_uint(__half2float(__ushort_as_half((unsigned short)h))); }

// ---- TMA bulk copies and mbarriers (as kernels.cu) ----
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar) { asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(smem_u32(bar)) : "memory"); }
__device__ __forceinline__ void bulk_g2s(void* s, const void* g, uint32_t bytes, uint64_t* bar) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               :: "r"(smem_u32(s)), "l"(g), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  } while (!ok);
}
template <bool EF>
__device__ __forceinline__ void bulk_s2g(void* g, const void* s, uint32_t bytes, uint64_t pol) {
  if (EF)
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;" :: "l"(g), "r"(smem_u32(s)), "r"(bytes), "l"(pol) : "memory");
  else
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" :: "l"(g), "r"(smem_u32(s)), "r"(bytes) : "memory");
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

extern __shared__ __align__(128) uint8_t smem[];

// ---------------------------------------------------------------- write-only
template <uint32_t R>
__global__ void __launch_bounds__(kT, 3) w_st(uint8_t* dst) {
  uint8_t* d = dst + (uint64_t)blockIdx.x * R * kRoundBytes;
  const uint4 v = make_uint4(threadIdx.x, blockIdx.x, 1, 2);
  for (uint32_t r = 0; r < R; ++r)
#pragma unroll
    for (uint32_t i = 0; i < 8; ++i) st_stream(d + r * kRoundBytes + 16u * (i * kT + threadIdx.x), v);
}
template <uint32_t R>
__global__ void __launch_bounds__(kT, 3) w_tma(uint8_t* dst) {
  uint8_t* d = dst + (uint64_t)blockIdx.x * R * kRoundBytes;
  uint4* s = reinterpret_cast<uint4*>(smem);
#pragma unroll
  for (uint32_t i = 0; i < 8; ++i) s[i * kT + threadIdx.x] = make_uint4(threadIdx.x, blockIdx.x, 1, 2);
  fence_async_smem();
  __syncthreads();
  if (threadIdx.x == 0) {
    for (uint32_t r = 0; r < R; ++r) bulk_s2g<false>(d + r * kRoundBytes, smem, kRoundBytes, 0);
    bulk_wait_all();
  }
}

// ---------------------------------------------------------------- read-only
template <uint32_t R>
__global__ void __launch_bounds__(kT, 3) r_ld(const uint8_t* src, uint32_t* sink) {
  const uint8_t* a = src + (uint64_t)blockIdx.x * R * kRoundBytes;
  uint32_t x = 0;
  for (uint32_t r = 0; r < R; ++r) {
    uint4 v[8];
#pragma unroll
    for (uint32_t i = 0; i < 8; ++i) v[i] = ld_stream(a + r * kRoundBytes + 16u * (i * kT + threadIdx.x));
#pragma unroll
    for (uint32_t i = 0; i < 8; ++i) x ^= v[i].x ^ v[i].y ^ v[i].z ^ v[i].w;
  }
  if (x == 0x9E3779B9u) sink[0] = x;
}
template <uint32_t R>
__global__ void __launch_bounds__(kT, 3) r_tma(const uint8_t* src, uint32_t* sink) {
  __shared__ __align__(8) uint64_t bar[2];
  const uint8_t* a = src + (uint64_t)blockIdx.x * R * kRoundBytes;
  if (threadIdx.x != 0) return;
  mbar_init(&bar[0]); mbar_init(&bar[1]);
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  for (uint32_t c = 0; c < 2 && c < R; ++c) bulk_g2s(smem + c * kRoundBytes, a + c * kRoundBytes, kRoundBytes, &bar[c]);
  for (uint32_t c = 0; c < R; ++c) {
    mbar_wait(&bar[c & 1], (c >> 1) & 1);
    if (c + 2 < R) bulk_g2s(smem + (c & 1) * kRoundBytes, a + (c + 2) * kRoundBytes, kRoundBytes, &bar[c & 1]);
  }
  const uint32_t x = reinterpret_cast<const uint32_t*>(smem)[0];
  if (x == 0x9E3779B9u) sink[0] = x;
}

// ---------------------------------------------------------------- 1:1 copy, registers in
// EF: st.global with an L2 evict-first policy
template <uint32_t R, bool EF>
__global__ void __launch_bounds__(kT, 3) c_reg_st(const uint8_t* src, uint8_t* dst) {
  const uint64_t t0 = (uint64_t)blockIdx.x * R * kRoundBytes;
  const uint64_t pol = EF ? evict_first_policy() : 0;
  for (uint32_t r = 0; r < R; ++r) {
    uint4 a[8];
#pragma unroll
    for (uint32_t i = 0; i < 8; ++i) a[i] = ld_stream(src + t0 + r * kRoundBytes + 16u * (i * kT + threadIdx.x));
#pragma unroll
    for (uint32_t i = 0; i < 8; ++i) {
      uint8_t* p = dst + t0 + r * kRoundBytes + 16u * (i * kT + threadIdx.x);
      if (EF) st_stream_hint(p, fix(a[i]), pol); else st_stream(p, fix(a[i]));
    }
  }
}
// registers in, two 32 KB shared out-buffers, one bulk store per round (the proposed move_kernel body)
template <uint32_t R, bool EF>
__global__ void __launch_bounds__(kT, 3) c_reg_tma(const uint8_t* src, uint8_t* dst) {
  const uint64_t t0 = (uint64_t)blockIdx.x * R * kRoundBytes;
  const uint64_t pol = EF ? evict_first_policy() : 0;
  for (uint32_t r = 0; r < R; ++r) {
    uint4 a[8];
#pragma unroll
    for (uint32_t i = 0; i < 8; ++i) a[i] = ld_stream(src + t0 + r * kRoundBytes + 16u * (i * kT + threadIdx.x));
    uint4* o = reinterpret_cast<uint4*>(smem + (r & 1) * kRoundBytes);
#pragma unroll
    for (uint32_t i = 0; i < 8; ++i) o[i * kT + threadIdx.x] = fix(a[i]);
    fence_async_smem();
    if (threadIdx.x == 0) bulk_wait_read0();   // store r-1 has read its buffer: round r+1 may overwrite it
    __syncthreads();
    if (threadIdx.x == 0) bulk_s2g<EF>(dst + t0 + r * kRoundBytes, o, kRoundBytes, pol);
  }
  if (threadIdx.x == 0) bulk_wait_all();
}

// ---------------------------------------------------------------- 1:1 copy, TMA in (staged decode shape)
// CH-byte chunks, two in-buffers; OB = 0: st.global from registers, OB = 1 / 2: shared out-buffers and bulk stores
template <uint32_t CH, uint32_t TILE, uint32_t OB, bool EF>
__global__ void __launch_bounds__(kT, 2) c_tma(const uint8_t* src, uint8_t* dst) {
  constexpr uint32_t NC = TILE / CH, NV = CH / 16;
  __shared__ __align__(8) uint64_t bar[2];
  const uint64_t t0 = (uint64_t)blockIdx.x * TILE;
  const uint64_t pol = EF ? evict_first_policy() : 0;
  uint8_t* in = smem;
  uint8_t* out = smem + 2 * CH;
  if (threadIdx.x == 0) {
    mbar_init(&bar[0]); mbar_init(&bar[1]);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    for (uint32_t c = 0; c < 2 && c < NC; ++c) bulk_g2s(in + c * CH, src + t0 + c * CH, CH, &bar[c]);
  }
  __syncthreads();
  for (uint32_t c = 0; c < NC; ++c) {
    const uint32_t b = c & 1;
    mbar_wait(&bar[b], (c >> 1) & 1);
    const uint4* iv = reinterpret_cast<const uint4*>(in + b * CH);
    if (OB == 0) {
      for (uint32_t v = threadIdx.x; v < NV; v += kT) {
        uint8_t* p = dst + t0 + (uint64_t)c * CH + 16u * v;
        if (EF) st_stream_hint(p, fix(iv[v]), pol); else st_stream(p, fix(iv[v]));
      }
      __syncthreads();
    } else {
      if (OB == 1 && c > 0) {   // the one out-buffer: wait until the previous store has read it
        if (threadIdx.x == 0) bulk_wait_read0();
        __syncthreads();
      }
      uint4* ov = reinterpret_cast<uint4*>(out + (OB == 1 ? 0 : b * CH));
      for (uint32_t v = threadIdx.x; v < NV; v += kT) ov[v] = fix(iv[v]);
      fence_async_smem();
      if (OB == 2 && threadIdx.x == 0) bulk_wait_read0();
      __syncthreads();
      if (threadIdx.x == 0) bulk_s2g<EF>(dst + t0 + (uint64_t)c * CH, ov, CH, pol);
    }
    if (threadIdx.x == 0 && c + 2 < NC) bulk_g2s(in + b * CH, src + t0 + (uint64_t)(c + 2) * CH, CH, &bar[b]);
  }
  if (OB && threadIdx.x == 0) bulk_wait_all();
}

// ---------------------------------------------------------------- 1:2 widen (fp16 -> fp32)
template <uint32_t R>
__global__ void __launch_bounds__(kT, 3) wd_reg(const uint8_t* src, uint8_t* dst) {   // body_widen: 8 units of 16 B per thread per round
  const uint64_t s0 = (uint64_t)blockIdx.x * R * kRoundBytes;
  for (uint32_t r = 0; r < R; ++r) {
    uint4 h[8];
#pragma unroll
    for (uint32_t i = 0; i < 8; ++i) h[i] = ld_stream(src + s0 + r * kRoundBytes + 16u * (i * kT + threadIdx.x));
#pragma unroll
    for (uint32_t i = 0; i < 8; ++i) {
      const uint4 x = h[i];
      const uint4 lo = make_uint4(widen(x.x & 0xFFFF), widen(x.x >> 16), widen(x.y & 0xFFFF), widen(x.y >> 16));
      const uint4 hi = make_uint4(widen(x.z & 0xFFFF), widen(x.z >> 16), widen(x.w & 0xFFFF), widen(x.w >> 16));
      uint8_t* p = dst + 2 * (s0 + r * kRoundBytes) + 32u * (i * kT + threadIdx.x);
      st_stream(p, lo); st_stream(p + 16, hi);
    }
  }
}
// TMA in (16 KB chunks, two buffers), widen into a 32 KB out-buffer (two), bulk store
template <uint32_t TILE>
__global__ void __launch_bounds__(kT, 2) wd_tma(const uint8_t* src, uint8_t* dst) {
  constexpr uint32_t CH = 16384, NC = TILE / CH, NU = CH / 16;
  __shared__ __align__(8) uint64_t bar[2];
  const uint64_t s0 = (uint64_t)blockIdx.x * TILE;
  uint8_t* in = smem;
  uint8_t* out = smem + 2 * CH;
  if (threadIdx.x == 0) {
    mbar_init(&bar[0]); mbar_init(&bar[1]);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    for (uint32_t c = 0; c < 2 && c < NC; ++c) bulk_g2s(in + c * CH, src + s0 + c * CH, CH, &bar[c]);
  }
  __syncthreads();
  for (uint32_t c = 0; c < NC; ++c) {
    const uint32_t b = c & 1;
    mbar_wait(&bar[b], (c >> 1) & 1);
    const uint4* iv = reinterpret_cast<const uint4*>(in + b * CH);
    uint4* ov = reinterpret_cast<uint4*>(out + b * 2 * CH);
    for (uint32_t u = threadIdx.x; u < NU; u += kT) {
      const uint4 x = iv[u];
      ov[2 * u] = make_uint4(widen(x.x & 0xFFFF), widen(x.x >> 16), widen(x.y & 0xFFFF), widen(x.y >> 16));
      ov[2 * u + 1] = make_uint4(widen(x.z & 0xFFFF), widen(x.z >> 16), widen(x.w & 0xFFFF), widen(x.w >> 16));
    }
    fence_async_smem();
    if (threadIdx.x == 0) bulk_wait_read0();
    __syncthreads();
    if (threadIdx.x == 0) {
      bulk_s2g<false>(dst + 2 * (s0 + (uint64_t)c * CH), ov, 2 * CH, 0);
      if (c + 2 < NC) bulk_g2s(in + b * CH, src + s0 + (uint64_t)(c + 2) * CH, CH, &bar[b]);
    }
  }
  if (threadIdx.x == 0) bulk_wait_all();
}

// ---------------------------------------------------------------- checks
__global__ void fill_src(uint32_t* p, uint64_t n) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
    p[i] = (uint32_t)(i * 2654435761u) & 0x3FFFFFFFu;   // finite floats / halfs: the fix-up leaves them alone
}
__global__ void count_diff(const uint32_t* a, const uint32_t* b, uint64_t n, unsigned long long* bad) {
  unsigned long long k = 0;
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) k += a[i] != b[i];
  if (k) atomicAdd(bad, k);
}
__global__ void count_widen_diff(const uint16_t* h, const uint32_t* f, uint64_t n, unsigned long long* bad) {
  unsigned long long k = 0;
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) k += widen(h[i]) != f[i];
  if (k) atomicAdd(bad, k);
}

// ---------------------------------------------------------------- driver
struct Variant {
  std::string group, name;
  double bytes;                      // read + write per launch
  std::function<void(cudaStream_t)> launch;
  std::function<long long()> check;  // mismatching words after a launch, -1: nothing to check
  int occ;                           // CTAs per SM the occupancy API reports
  std::vector<double> gbs;
};

static uint32_t pad_for(int ctas_per_sm) {   // dynamic shared memory that leaves room for exactly this many CTAs per SM
  return ctas_per_sm == 1 ? 120u << 10 : ctas_per_sm == 2 ? 80u << 10 : 58u << 10;
}

int main(int argc, char** argv) {
  const int runs = argc > 1 ? atoi(argv[1]) : 3;
  const int launches = argc > 2 ? atoi(argv[2]) : 20;
  const uint64_t N = 1ull << 30;
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  printf("%s, %d SMs, %zu KB shared memory per SM; 1 GiB per launch, %d launches x %d runs\n", prop.name, prop.multiProcessorCount,
         prop.sharedMemPerMultiprocessor >> 10, launches, runs);
  uint8_t *src, *dst;
  unsigned long long* bad;
  uint32_t* sink;
  CK(cudaMalloc(&src, N)); CK(cudaMalloc(&dst, N)); CK(cudaMalloc(&bad, 8)); CK(cudaMalloc(&sink, 4));
  cudaStream_t st;
  CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  fill_src<<<1024, 256, 0, st>>>((uint32_t*)src, N / 4);
  CK(cudaStreamSynchronize(st));

  auto check_copy = [&]() -> long long {
    CK(cudaMemsetAsync(bad, 0, 8, st));
    count_diff<<<1024, 256, 0, st>>>((const uint32_t*)src, (const uint32_t*)dst, N / 4, bad);
    unsigned long long h; CK(cudaMemcpyAsync(&h, bad, 8, cudaMemcpyDeviceToHost, st)); CK(cudaStreamSynchronize(st));
    return (long long)h;
  };
  auto check_widen = [&]() -> long long {
    CK(cudaMemsetAsync(bad, 0, 8, st));
    count_widen_diff<<<1024, 256, 0, st>>>((const uint16_t*)src, (const uint32_t*)dst, N / 4, bad);
    unsigned long long h; CK(cudaMemcpyAsync(&h, bad, 8, cudaMemcpyDeviceToHost, st)); CK(cudaStreamSynchronize(st));
    return (long long)h;
  };
  auto none = []() -> long long { return -1; };

  std::vector<Variant> V;
  // a kernel launch with `need` bytes of dynamic shared memory, padded to `ctas` CTAs per SM
  auto add = [&](const char* group, std::string name, double bytes, auto kern, uint32_t grid, uint32_t need, int ctas,
                 std::function<long long()> check, auto... args) {
    const uint32_t dyn = std::max(need, pad_for(ctas));
    // the largest size any launch of this kernel asks for (the attribute is per kernel, not per launch)
    CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pad_for(1)));
    int occ = 0;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, kT, dyn));
    V.push_back({group, name + " @" + std::to_string(ctas) + "/SM", bytes,
                 [=](cudaStream_t s) { kern<<<grid, kT, dyn, s>>>(args...); }, check, occ, {}});
  };
  const uint32_t g64 = (uint32_t)(N / 65536), g256 = (uint32_t)(N / 262144);
  const double W = (double)N, C = 2.0 * N, Wd = 1.5 * N;   // write-only, copy, widen (N/2 read, N written)

  V.push_back({"write", "cudaMemsetAsync", W, [=](cudaStream_t s) { CK(cudaMemsetAsync(dst, 0, N, s)); }, none, 0, {}});
  add("write", "st.global.v4 (regs, 64 KB tiles)", W, w_st<2>, g64, 0, 3, none, dst);
  add("write", "TMA bulk store (32 KB smem, 64 KB tiles)", W, w_tma<2>, g64, kRoundBytes, 3, none, dst);
  add("read", "ld.global.nc.v4 + xor (64 KB tiles)", W, r_ld<2>, g64, 0, 3, none, (const uint8_t*)src, sink);
  add("read", "TMA bulk load (2 x 32 KB, 256 KB tiles)", W, r_tma<8>, g256, 2 * kRoundBytes, 2, none, (const uint8_t*)src, sink);
  for (int k = 1; k <= 3; ++k) {
    add("copy", "reg in, st.global out (move_kernel)", C, c_reg_st<2, false>, g64, 0, k, check_copy, (const uint8_t*)src, dst);
    add("copy", "reg in, st.global evict-first out", C, c_reg_st<2, true>, g64, 0, k, check_copy, (const uint8_t*)src, dst);
    add("copy", "reg in, TMA out (2 x 32 KB)", C, c_reg_tma<2, false>, g64, 2 * kRoundBytes, k, check_copy, (const uint8_t*)src, dst);
    add("copy", "reg in, TMA evict-first out (2 x 32 KB)", C, c_reg_tma<2, true>, g64, 2 * kRoundBytes, k, check_copy, (const uint8_t*)src, dst);
  }
  for (int k = 1; k <= 3; ++k) {
    if (k < 3) {   // 2 x 32 KB in (+ 32 KB out) does not fit three times
      add("copy", "TMA in 2x32K, st.global out (staged decode)", C, c_tma<32768, 262144, 0, false>, g256, 2 * 32768, k, check_copy,
          (const uint8_t*)src, dst);
      add("copy", "TMA in 2x32K, TMA out 1x32K", C, c_tma<32768, 262144, 1, false>, g256, 3 * 32768, k, check_copy, (const uint8_t*)src, dst);
      add("copy", "TMA in 2x32K, TMA evict-first out 1x32K", C, c_tma<32768, 262144, 1, true>, g256, 3 * 32768, k, check_copy,
          (const uint8_t*)src, dst);
    }
    add("copy", "TMA in 2x16K, st.global out", C, c_tma<16384, 262144, 0, false>, g256, 2 * 16384, k, check_copy, (const uint8_t*)src, dst);
    add("copy", "TMA in 2x16K, TMA out 2x16K", C, c_tma<16384, 262144, 2, false>, g256, 4 * 16384, k, check_copy, (const uint8_t*)src, dst);
    add("copy", "TMA in 2x16K, TMA evict-first out 2x16K", C, c_tma<16384, 262144, 2, true>, g256, 4 * 16384, k, check_copy,
        (const uint8_t*)src, dst);
  }
  for (int k = 1; k <= 2; ++k) {
    add("widen", "body_widen: reg in, st.global out", Wd, wd_reg<1>, (uint32_t)(N / 2 / 32768), 0, k, check_widen, (const uint8_t*)src, dst);
    add("widen", "TMA in 2x16K, widen in smem, TMA out 2x32K", Wd, wd_tma<131072>, (uint32_t)(N / 2 / 131072), 6 * 16384, k, check_widen,
        (const uint8_t*)src, dst);
  }
  add("widen", "body_widen: reg in, st.global out", Wd, wd_reg<1>, (uint32_t)(N / 2 / 32768), 0, 3, check_widen, (const uint8_t*)src, dst);

  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  for (int run = 0; run < runs; ++run) {
    for (auto& v : V) {
      for (int w = 0; w < 3; ++w) v.launch(st);
      CK(cudaGetLastError());
      CK(cudaStreamSynchronize(st));
      CK(cudaEventRecord(e0, st));
      for (int l = 0; l < launches; ++l) v.launch(st);
      CK(cudaEventRecord(e1, st));
      CK(cudaEventSynchronize(e1));
      float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
      v.gbs.push_back(v.bytes * launches / (ms * 1e-3) / 1e9);
      if (run == 0) {
        const long long b = v.check();
        if (b > 0) { printf("MISMATCH: %s: %lld words differ\n", v.name.c_str(), b); return 1; }
      }
    }
  }
  printf("\n| group | variant | CTAs/SM (occupancy API) | GB/s r+w, median of %d | runs |\n|---|---|---|---|---|\n", runs);
  for (auto& v : V) {
    std::vector<double> s = v.gbs;
    std::sort(s.begin(), s.end());
    std::string all;
    for (double g : v.gbs) { char b[32]; snprintf(b, sizeof b, "%s%.0f", all.empty() ? "" : " ", g); all += b; }
    printf("| %s | %s | %s | %.0f | %s |\n", v.group.c_str(), v.name.c_str(), v.occ ? std::to_string(v.occ).c_str() : "-", s[s.size() / 2],
           all.c_str());
  }
  return 0;
}
