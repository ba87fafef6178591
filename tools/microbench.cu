// microbench.cu - design-space probe for the 4 MiB pack kernel (NOT part of the product).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -o build/microbench tools/microbench.cu
// Each variant copies P bytes src->dst (dst shifted by `shift` bytes) rotating through a ring > L2, and is
// timed (a) eagerly back-to-back and (b) as a CUDA graph of ring-many launches; ncu gives per-launch time.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <vector>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); exit(1); } } while (0)

__device__ __forceinline__ uint4 ld_stream(const uint4* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ void st_stream(uint4* p, uint4 v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" :: "l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ uint32_t q(uint32_t w) { return ((w & 0x7FFFFFFFu) > 0x7F800000u) ? (w | 0x00400000u) : w; }
__device__ __forceinline__ uint4 fix(uint4 v) { v.x = q(v.x); v.y = q(v.y); v.z = q(v.z); v.w = q(v.w); return v; }

// V vectors per thread, blocked by CTA: CTA b covers vectors [b*T*V, (b+1)*T*V), thread t takes t, t+T, ...
template <int V>
__global__ void copy_simple(const uint4* __restrict__ src, uint4* __restrict__ dst, uint32_t nvec) {
  const uint32_t T = blockDim.x;
  const uint32_t base = blockIdx.x * T * V + threadIdx.x;
  uint4 a[V];
#pragma unroll
  for (int i = 0; i < V; ++i) if (base + i * T < nvec) a[i] = ld_stream(src + base + i * T);
#pragma unroll
  for (int i = 0; i < V; ++i) if (base + i * T < nvec) st_stream(dst + base + i * T, fix(a[i]));
}

// header bytes passed by value + payload copy: the shape of the C2 encode
struct Hdr { uint8_t b[64]; uint32_t n; };
template <int V>
__global__ void copy_hdr(const uint4* __restrict__ src, uint8_t* __restrict__ wire, uint32_t nvec, const __grid_constant__ Hdr h, uint32_t pad) {
  const uint32_t T = blockDim.x;
  if (blockIdx.x == 0 && threadIdx.x < h.n) wire[pad + threadIdx.x] = h.b[threadIdx.x];
  uint4* dst = reinterpret_cast<uint4*>(wire + pad + h.n);
  const uint32_t base = blockIdx.x * T * V + threadIdx.x;
  uint4 a[V];
#pragma unroll
  for (int i = 0; i < V; ++i) if (base + i * T < nvec) a[i] = ld_stream(src + base + i * T);
#pragma unroll
  for (int i = 0; i < V; ++i) if (base + i * T < nvec) st_stream(dst + base + i * T, fix(a[i]));
}

// persistent-style: grid = k * SMs, grid-stride loop with 4-way unroll
__global__ void copy_gridstride(const uint4* __restrict__ src, uint4* __restrict__ dst, uint32_t nvec) {
  const uint32_t stride = gridDim.x * blockDim.x;
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  for (; i + 3 * stride < nvec; i += 4 * stride) {
    uint4 a = ld_stream(src + i), b = ld_stream(src + i + stride), c = ld_stream(src + i + 2 * stride), d = ld_stream(src + i + 3 * stride);
    st_stream(dst + i, fix(a)); st_stream(dst + i + stride, fix(b)); st_stream(dst + i + 2 * stride, fix(c)); st_stream(dst + i + 3 * stride, fix(d));
  }
  for (; i < nvec; i += stride) st_stream(dst + i, fix(ld_stream(src + i)));
}

// TMA bulk: one elected thread per CTA moves CH bytes global->smem->global (raw copy, no fix-up)
template <int CH>
__global__ void copy_bulk(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, uint32_t nbytes) {
  extern __shared__ __align__(128) uint8_t sm[];
  __shared__ __align__(8) uint64_t bar;
  const uint32_t off = blockIdx.x * CH;
  if (off >= nbytes) return;
  const uint32_t n = min((uint32_t)CH, nbytes - off);
  if (threadIdx.x == 0) {
    uint32_t b = (uint32_t)__cvta_generic_to_shared(&bar), s = (uint32_t)__cvta_generic_to_shared(sm);
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(b));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(b), "r"(n) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(s), "l"(src + off), "r"(n), "r"(b) : "memory");
    uint32_t done = 0;
    while (!done) {
      asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0; selp.u32 %0, 1, 0, p; }" : "=r"(done) : "r"(b) : "memory");
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" :: "l"(dst + off), "r"(s), "r"(n) : "memory");
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
  }
}

struct Ring { std::vector<uint8_t*> src, dst; };

template <typename F>
static void time_variant(const char* name, F launch, int ring, cudaStream_t st, double bytes) {
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  for (int i = 0; i < ring; ++i) launch(i);
  CK(cudaStreamSynchronize(st));
  const int reps = 10;
  CK(cudaEventRecord(e0, st));
  for (int r = 0; r < reps; ++r) for (int i = 0; i < ring; ++i) launch(i);
  CK(cudaEventRecord(e1, st));
  CK(cudaEventSynchronize(e1));
  float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
  double eager_us = ms * 1e3 / (reps * ring);
  // graph
  cudaGraph_t g; cudaGraphExec_t ge;
  CK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
  for (int i = 0; i < ring; ++i) launch(i);
  CK(cudaStreamEndCapture(st, &g));
  CK(cudaGraphInstantiate(&ge, g, 0));
  CK(cudaGraphLaunch(ge, st)); CK(cudaStreamSynchronize(st));
  CK(cudaEventRecord(e0, st));
  for (int r = 0; r < reps; ++r) CK(cudaGraphLaunch(ge, st));
  CK(cudaEventRecord(e1, st));
  CK(cudaEventSynchronize(e1));
  CK(cudaEventElapsedTime(&ms, e0, e1));
  double graph_us = ms * 1e3 / (reps * ring);
  printf("%-34s eager %7.2f us  graph %7.2f us  -> %7.1f GB/s (graph, r+w)\n", name, eager_us, graph_us, bytes / graph_us / 1e3);
  CK(cudaGraphExecDestroy(ge)); CK(cudaGraphDestroy(g));
}

int main(int argc, char** argv) {
  const uint32_t P = argc > 1 ? (uint32_t)atoi(argv[1]) : 4u << 20;
  const int ring = argc > 2 ? atoi(argv[2]) : 48;
  const uint32_t nvec = P / 16;
  cudaStream_t st; CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  Ring R;
  for (int i = 0; i < ring; ++i) {
    uint8_t *s, *d;
    CK(cudaMalloc(&s, P)); CK(cudaMalloc(&d, P + 4096));
    CK(cudaMemset(s, i + 1, P)); CK(cudaMemset(d, 0, P + 4096));
    R.src.push_back(s); R.dst.push_back(d);
  }
  CK(cudaDeviceSynchronize());
  const double bytes = 2.0 * P;
  printf("P = %u bytes, ring %d (%.0f MiB)\n", P, ring, ring * 2.0 * P / 1048576);
  time_variant("cudaMemcpyAsync D2D", [&](int i) { CK(cudaMemcpyAsync(R.dst[i], R.src[i], P, cudaMemcpyDeviceToDevice, st)); }, ring, st, bytes);
#define SIMPLE(V, T) time_variant("simple V=" #V " T=" #T, [&](int i) { \
    copy_simple<V><<<(nvec + (T) * (V) - 1) / ((T) * (V)), T, 0, st>>>((const uint4*)R.src[i], (uint4*)R.dst[i], nvec); }, ring, st, bytes)
  SIMPLE(1, 256); SIMPLE(1, 512); SIMPLE(1, 1024);
  SIMPLE(2, 256); SIMPLE(2, 512); SIMPLE(2, 1024);
  SIMPLE(4, 256); SIMPLE(4, 512); SIMPLE(4, 1024);
  SIMPLE(8, 256); SIMPLE(8, 512);
  Hdr h; h.n = 47; for (int k = 0; k < 64; ++k) h.b[k] = (uint8_t)k;
  const uint32_t pad = (128 - 47 % 128) % 128;
#define HDR(V, T) time_variant("hdr+copy V=" #V " T=" #T, [&](int i) { \
    copy_hdr<V><<<(nvec + (T) * (V) - 1) / ((T) * (V)), T, 0, st>>>((const uint4*)R.src[i], R.dst[i], nvec, h, pad); }, ring, st, bytes)
  HDR(1, 512); HDR(2, 512); HDR(4, 256);
  for (int k : {1, 2, 4, 8}) {
    char nm[64]; snprintf(nm, sizeof nm, "gridstride %dxSM T=512", k);
    time_variant(nm, [&](int i) { copy_gridstride<<<132 * k, 512, 0, st>>>((const uint4*)R.src[i], (uint4*)R.dst[i], nvec); }, ring, st, bytes);
  }
  for (int k : {2, 4}) {
    char nm[64]; snprintf(nm, sizeof nm, "gridstride %dxSM T=1024", k);
    time_variant(nm, [&](int i) { copy_gridstride<<<132 * k, 1024, 0, st>>>((const uint4*)R.src[i], (uint4*)R.dst[i], nvec); }, ring, st, bytes);
  }
  CK(cudaFuncSetAttribute(copy_bulk<32768>, cudaFuncAttributeMaxDynamicSharedMemorySize, 32768));
  CK(cudaFuncSetAttribute(copy_bulk<16384>, cudaFuncAttributeMaxDynamicSharedMemorySize, 16384));
  CK(cudaFuncSetAttribute(copy_bulk<8192>, cudaFuncAttributeMaxDynamicSharedMemorySize, 8192));
  time_variant("bulk(TMA) 32K/CTA", [&](int i) { copy_bulk<32768><<<(P + 32767) / 32768, 32, 32768, st>>>(R.src[i], R.dst[i], P); }, ring, st, bytes);
  time_variant("bulk(TMA) 16K/CTA", [&](int i) { copy_bulk<16384><<<(P + 16383) / 16384, 32, 16384, st>>>(R.src[i], R.dst[i], P); }, ring, st, bytes);
  time_variant("bulk(TMA) 8K/CTA", [&](int i) { copy_bulk<8192><<<(P + 8191) / 8192, 32, 8192, st>>>(R.src[i], R.dst[i], P); }, ring, st, bytes);
  // correctness spot check of the last variant
  std::vector<uint8_t> hb(64);
  CK(cudaMemcpy(hb.data(), R.dst[0] + P - 64, 64, cudaMemcpyDeviceToHost));
  printf("tail byte %u (expect 1)\n", hb[63]);
  return 0;
}
