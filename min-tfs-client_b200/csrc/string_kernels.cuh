// string_kernels.cuh - DT_STRING keys of the concatenated batch decode as offset-indexed byte columns (plan.h StrTables; the host
// side is b200tfs_decode_concat_strings in codec_host.cpp, the walk is string_walk.h).  Included by kernels.cu inside namespace
// b200tfs, after concat_plan_strings_kernel, which has placed every (record, string key)'s n_strings offset entries.  Launch order,
// no host step between them:
//   str_index_kernel  a warp per pair: its lane 0 walks the pair's TensorProto with the record's cursor and packs, for string j,
//                     (record-relative wire offset << 32 | byte position within the pair's strings) into offset entry j; the
//                     pair's byte total goes to T.bytes.  A walk that finds another count than the parse (a map entry that
//                     carries its TensorProto in several `value` occurrences) marks the pair B200TFS_E_NONCANONICAL, and never
//                     writes past the n_strings entries the plan reserved.
//   str_scan_kernel   one CTA: per key, a block scan of the byte totals gives each pair its first data byte (B200TFS_E_SIZE past
//                     data_cap) and the chunks of kStrChunk strings their numbers; offsets[m] behind the key's last OK pair
//   str_copy_kernel   a warp per chunk, striding: a lane per string of at most kStrLaneCopy bytes, the warp for longer ones
//                     (warp_copy_strings, strcol.h)
//   str_fix_kernel    the same chunks: every entry becomes its string's first byte in the key's data.  Separate from the copy,
//                     which reads the entry behind each string for its length.

// The index kernels' sink (walk_strings): string j's entry goes to slot[place(j)] - here entry j; the padded decode's index kernel
// (padded_kernels.cuh) places it at its padded position.
struct StrPlaceSame {
  __device__ __forceinline__ uint64_t operator()(uint64_t j) const { return j; }
};
template <class Place = StrPlaceSame>
struct StrIndexSink {
  uint64_t* slot;
  uint64_t cap;   // strings the plan reserved entries for (n_strings)
  uint32_t pos;   // bytes of the strings so far
  Place place;
  __device__ __forceinline__ void operator()(uint64_t j, uint32_t off, uint32_t len) {
    if (j < cap) slot[place(j)] = ((uint64_t)off << 32) | pos;
    pos += len;
  }
};

__global__ void __launch_bounds__(kStrThreads) str_index_kernel(const __grid_constant__ StrTables T) {
  __shared__ __align__(16) uint8_t lines[kStrThreads / 32][256];
  const uint32_t warp = threadIdx.x >> 5;
  const uint64_t p = (uint64_t)blockIdx.x * (kStrThreads / 32) + warp;   // pair r * n_keys + k
  if (p >= (uint64_t)T.n * T.n_keys || (threadIdx.x & 31)) return;
  const uint32_t r = (uint32_t)(p / T.n_keys), k = (uint32_t)(p % T.n_keys);
  b200tfs_output& o = T.vouts[(size_t)r * kFusedMaxOutputs + k];
  uint64_t total = 0;
  if (o.status == B200TFS_OK && dtype_info(o.dtype).kind == VK_STRING) {
    Cursor c;
    cur_open(c, T.w + T.rec_off[r], (uint32_t)T.rec_len[r], lines[warp]);
    c.p = (uint32_t)o.msg_off;
    c.end = (uint32_t)(o.msg_off + o.msg_len);
    StrIndexSink<> sink{reinterpret_cast<uint64_t*>((uintptr_t)o.dst_off), o.n_strings, 0u, {}};
    const uint64_t found = walk_strings(c, sink);
    if (c.err || found != o.n_strings) o.status = B200TFS_E_NONCANONICAL;
    else total = sink.pos;
  }
  T.bytes[(size_t)k * T.n + r] = total;
}

__global__ void __launch_bounds__(kConcatPlanThreads) str_scan_kernel(const __grid_constant__ StrTables T) {
  __shared__ unsigned long long warp_sum[kConcatPlanThreads / 32];
  __shared__ int32_t last;
  const uint32_t n = T.n;
  uint64_t chunk_carry = 0;
  for (uint32_t k = 0; k < T.n_keys; ++k) {
    if (threadIdx.x == 0) last = -1;
    uint64_t byte_carry = 0;
    for (uint32_t r0 = 0; r0 < n; r0 += kConcatPlanThreads) {      // uniform trip count: the scans have barriers inside
      const uint32_t r = r0 + threadIdx.x;
      b200tfs_output* o = nullptr;
      bool ok = false;
      uint64_t b = 0;
      if (r < n) {
        o = &T.vouts[(size_t)r * kFusedMaxOutputs + k];
        ok = o->status == B200TFS_OK && dtype_info(o->dtype).kind == VK_STRING;
        if (ok) b = T.bytes[(size_t)k * n + r];
      }
      const uint64_t at = concat_scan(b, byte_carry, warp_sum);
      if (ok && at + b > T.keys[k].cap) { o->status = B200TFS_E_SIZE; ok = false; }
      const uint64_t chunks = ok ? (o->n_strings + kStrChunk - 1) / kStrChunk : 0;
      const uint64_t c0 = concat_scan(chunks, chunk_carry, warp_sum);
      if (r < n) {
        T.data0[(size_t)k * n + r] = at;
        T.chunk0[(size_t)k * n + r] = c0;
        if (ok) atomicMax(&last, (int32_t)r);
      }
    }
    __syncthreads();
    if (threadIdx.x == 0 && last >= 0) {   // offsets[m]: inside dst_cap, which the plan checked for the entry behind every pair
      const b200tfs_output& o = T.vouts[(size_t)last * kFusedMaxOutputs + k];
      const size_t q = (size_t)k * n + (uint32_t)last;
      reinterpret_cast<uint64_t*>((uintptr_t)o.dst_off)[o.n_strings] = T.data0[q] + T.bytes[q];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) *T.n_chunks = chunk_carry;
}

// the pair (k * n + r) that copy chunk c belongs to: the last one whose first chunk is at or before c
__device__ __forceinline__ uint64_t str_pair_of(const StrTables& T, uint64_t c) {
  uint64_t lo = 0, hi = (uint64_t)T.n * T.n_keys;
#pragma unroll 1
  while (hi - lo > 1) {
    const uint64_t mid = (lo + hi) >> 1;
    if (T.chunk0[mid] <= c) lo = mid; else hi = mid;
  }
  return lo;
}

__global__ void __launch_bounds__(kStrThreads) str_copy_kernel(const __grid_constant__ StrTables T) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t total = *T.n_chunks, nw = ((uint64_t)gridDim.x * kStrThreads) >> 5;
#pragma unroll 1
  for (uint64_t c = ((uint64_t)blockIdx.x * kStrThreads + threadIdx.x) >> 5; c < total; c += nw) {   // warp-uniform
    const uint64_t q = str_pair_of(T, c);
    const uint32_t k = (uint32_t)(q / T.n), r = (uint32_t)(q % T.n);
    const b200tfs_output& o = T.vouts[(size_t)r * kFusedMaxOutputs + k];
    const uint64_t* slot = reinterpret_cast<const uint64_t*>((uintptr_t)o.dst_off);
    const uint8_t* rec = T.w + T.rec_off[r];
    uint8_t* dst = T.keys[k].data + T.data0[q];
    const uint64_t cnt = o.n_strings, j0 = (c - T.chunk0[q]) * kStrChunk;
    const uint32_t end = (uint32_t)T.bytes[q];
#pragma unroll 1
    for (uint32_t i = 0; i < kStrChunk && j0 + i < cnt; i += 32) {
      const uint64_t j = j0 + i + lane;
      uint32_t src = 0, pos = 0, len = 0;
      if (j < cnt) {
        const uint64_t e = slot[j];
        src = (uint32_t)(e >> 32);
        pos = (uint32_t)e;
        len = (j + 1 < cnt ? (uint32_t)slot[j + 1] : end) - pos;
      }
      warp_copy_strings(dst + pos, rec + src, len, j < cnt, UINT64_MAX);
    }
  }
}

__global__ void __launch_bounds__(kStrThreads) str_fix_kernel(const __grid_constant__ StrTables T) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t total = *T.n_chunks, nw = ((uint64_t)gridDim.x * kStrThreads) >> 5;
#pragma unroll 1
  for (uint64_t c = ((uint64_t)blockIdx.x * kStrThreads + threadIdx.x) >> 5; c < total; c += nw) {
    const uint64_t q = str_pair_of(T, c);
    const uint32_t k = (uint32_t)(q / T.n), r = (uint32_t)(q % T.n);
    const b200tfs_output& o = T.vouts[(size_t)r * kFusedMaxOutputs + k];
    uint64_t* slot = reinterpret_cast<uint64_t*>((uintptr_t)o.dst_off);
    const uint64_t cnt = o.n_strings, j0 = (c - T.chunk0[q]) * kStrChunk, base = T.data0[q];
#pragma unroll 1
    for (uint64_t j = j0 + lane; j < j0 + kStrChunk && j < cnt; j += 32) slot[j] = base + (uint32_t)slot[j];
  }
}

cudaError_t launch_concat_strings(const StrTables& T, uint32_t grid, cudaStream_t stream) {
  const uint64_t pairs = (uint64_t)T.n * T.n_keys, per = kStrThreads / 32;
  str_index_kernel<<<(uint32_t)((pairs + per - 1) / per), kStrThreads, 0, stream>>>(T);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  str_scan_kernel<<<1, kConcatPlanThreads, 0, stream>>>(T);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  str_copy_kernel<<<std::max(1u, grid), kStrThreads, 0, stream>>>(T);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  str_fix_kernel<<<std::max(1u, grid), kStrThreads, 0, stream>>>(T);
  return cudaGetLastError();
}
