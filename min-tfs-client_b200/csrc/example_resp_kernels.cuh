// example_resp_kernels.cuh - Classify / Regress responses: a batch of responses into one value / score array (plan.h XrTables;
// planned by example_host.inc; the walk is example_walk.h).  Included by kernels.cu inside namespace b200tfs, after concat_scan.
//
//   xr_index_kernel    one warp per response: lane 0 walks the top level and the model_spec, the whole warp finds the entries
//                      of every `result` body a 256-byte window at a time (xr_warp_entries) and writes their {off, len} into
//                      the response's slots; Classify: it also counts the classes of the response's first example
//   xr_scan_kernel     one CTA: the first row of every response (block scan of the row counts), C (the class count of the batch's
//                      first example), B200TFS_E_SIZE for a response whose rows end past a capacity
//   xr_emit_kernel     one thread per row, striding: Regress reads a canonical entry (`0D f32`, or empty) directly and walks any
//                      other; Classify walks the example's classes and stores score and label reference of every class c < C
//   xr_compare_kernel  Classify: one warp per row compares its labels with the first example's; a difference clears same_labels
//   xr_publish_kernel  one CTA: per-response and batch results to pinned memory
//
// What the reference does here: ClassificationResponse.FromString / RegressionResponse.FromString (prediction_service_pb2_grpc.py)
// and a Python loop over every Classifications / Class / Regression message.

__device__ __forceinline__ void xr_prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

// xr_classes' sink for row `row`: scores and label references of the classes c < C, never at or past a capacity
struct XrClassSink {
  uint32_t* values; b200tfs_label_ref* labels;
  uint64_t base, C, values_cap, labels_cap;
  B2_HD void operator()(uint32_t k, uint32_t off, uint32_t len, uint32_t score) {
    if (k >= C) return;
    const uint64_t i = base + k;
    if (i < values_cap) values[i] = score;
    if (i < labels_cap) labels[i] = b200tfs_label_ref{off, len};
  }
};

// ---- the warp's entry finder ----------------------------------------------------------------------------------------------
// A message body is walked a window of kXrWin byte positions at a time.  Every lane works out, for each of its 8 positions,
// where a field starting there would end (xr_field_end: the checks of walker.h's rd_tag / rd_len / skip_scalar, on bytes staged
// in shared memory); pointer doubling over those ends (log2 kXrWin rounds) then marks the chain of field starts from the window's
// first position, and the chain's last member says where the next window starts.  A window costs the same for a hundred 2-byte
// entries as for one, and finding an entry never waits on a global load: the body is staged kXrStage bytes at a time.
constexpr uint32_t kXrWin = 256;
constexpr uint32_t kXrStage = 4096;
constexpr int32_t kXrErr = -1, kXrGroup = -2;
struct __align__(16) XrWarpSmem {   // 16-byte aligned: the staging stores are 128-bit vectors
  uint8_t buf[kXrStage];           // the staged bytes [gb, gb + kXrStage) of the record
  int32_t J[2][kXrWin];            // jump table of the doubling rounds (window-relative ends)
  int32_t nx[kXrWin];              // where the field at each position ends (window-relative), kXrErr, kXrGroup
  uint32_t bo[kXrWin], bl[kXrWin]; // the entry body of each position (bl = ~0u: not an entry)
  uint8_t M[kXrWin];               // on the chain
  int32_t exit_k, exit_t;          // the chain's last member in the window and where it ends
};

// rd_varint on staged bytes, without a loop: the bytes of the varint at b (0: it runs past `avail` bytes or over ten), its
// value in *v (bits past 64 fall off).  The ten loads are independent, so a lane that meets a long varint costs the warp little.
__device__ __forceinline__ uint32_t xr_varint(const uint8_t* b, uint32_t avail, uint64_t* v) {
  uint64_t x = 0;
  uint32_t n = 0;
#pragma unroll
  for (uint32_t i = 0; i < 10; ++i) {
    const uint32_t c = i < avail ? b[i] : 0x80u;
    if (!n) {
      x |= (uint64_t)(c & 0x7F) << (7 * i);
      if (!(c & 0x80)) n = i + 1;
    }
  }
  *v = x;
  return n;
}

// The field starting at byte b (record offset p, p < hi) of a body ending at hi: its end, kXrErr when malformed, kXrGroup for a
// start-group (skipped by the cursor).  A field-1 sub-message (an entry) also gets its body in *body / *blen.
__device__ __forceinline__ int64_t xr_field_end(const uint8_t* b, uint32_t p, uint32_t hi, uint32_t* body, uint32_t* blen) {
  const uint32_t avail = hi - p;
  if (avail >= 2 && !((b[0] | b[1]) & 0x80)) {             // one-byte tag, one-byte length or varint: what a server writes
    const uint32_t t0 = b[0], wt0 = t0 & 7;
    if ((t0 >> 3) == 0) return kXrErr;
    if (wt0 == WT_VARINT) return (int64_t)p + 2;
    if (wt0 == WT_LEN) {
      if (b[1] > avail - 2) return kXrErr;
      if (t0 == tag_of(1, WT_LEN)) { *body = p + 2; *blen = b[1]; }
      return (int64_t)p + 2 + b[1];
    }
  }
  uint64_t t, v;
  const uint32_t i = xr_varint(b, avail, &t);
  if (!i) return kXrErr;
  if (t > 0xFFFFFFFFull || (t >> 3) == 0) return kXrErr;   // rd_tag
  const uint32_t wt = (uint32_t)t & 7;
  if (wt == WT_I64) return avail - i < 8 ? kXrErr : (int64_t)p + i + 8;
  if (wt == WT_I32) return avail - i < 4 ? kXrErr : (int64_t)p + i + 4;
  if (wt == WT_SGROUP) return kXrGroup;
  if (wt != WT_VARINT && wt != WT_LEN) return kXrErr;      // stray END_GROUP, wire types 6 and 7
  const uint32_t i2 = xr_varint(b + i, avail - i, &v);
  if (!i2) return kXrErr;
  if (wt == WT_VARINT) return (int64_t)p + i + i2;
  if (v > 0x7FFFFFFFull || v > avail - i - i2) return kXrErr;   // rd_len
  if (t == tag_of(1, WT_LEN)) { *body = p + i + i2; *blen = (uint32_t)v; }
  return (int64_t)p + i + i2 + v;
}

// Stage record bytes from `from` on (16-byte vectors, never past the record's last vector)
__device__ __forceinline__ const uint8_t* xr_stage(XrWarpSmem& S, const uint8_t* from, const uint8_t* rend) {
  const uint8_t* gb = reinterpret_cast<const uint8_t*>((uintptr_t)from & ~(uintptr_t)15);
  const uint32_t lane = threadIdx.x & 31;
  __syncwarp();
  for (uint32_t v = lane; v < kXrStage / 16 && gb + 16 * v < rend; v += 32)
    reinterpret_cast<uint4*>(S.buf)[v] = reinterpret_cast<const uint4*>(gb)[v];
  __syncwarp();
  return gb;
}

// The entries (field-1 sub-messages) of the body [lo, hi) of the record rec[0, rec_len), found by the whole warp: entry i goes to
// slot[base + i] while base + i < cap (slot == nullptr: count only).  Returns how many there are; *err = B200TFS_E_PARSE when a
// field on the chain is malformed (what xr_entries reports).  Lane 0's cursor c, bound to the record, skips groups.
__device__ uint32_t xr_warp_entries(XrWarpSmem& S, Cursor& c, const uint8_t* rec, uint32_t rec_len, uint32_t lo, uint32_t hi,
                                    b200tfs_label_ref* slot, uint32_t base, uint32_t cap, int* err) {
  const uint32_t lane = threadIdx.x & 31;
  const uint8_t* rend = rec + rec_len;
  const uint8_t* gb = nullptr;
  uint32_t count = 0, s = lo;
  *err = 0;
#pragma unroll 1
  while (s < hi) {
    const uint32_t L = min(kXrWin, hi - s);
    const uint32_t need = min(hi, s + kXrWin + 32);        // a field at the window's last position reads at most 20 bytes
    if (!gb || rec + need > gb + kXrStage) gb = xr_stage(S, rec + s, rend);
    // kept in shared memory rather than registers: the loop stays rolled, and the kernel small enough for the instruction cache
#pragma unroll 1
    for (int j = 0; j < 8; ++j) {
      const uint32_t k = 32 * j + lane;
      uint32_t bo = 0, bl = ~0u;
      int32_t nx = (int32_t)L;
      if (k < L) {
        const int64_t e = xr_field_end(S.buf + (rec + s + k - gb), s + k, hi, &bo, &bl);
        nx = e < 0 ? (int32_t)e : (int32_t)(e - s);
      }
      S.nx[k] = nx; S.bo[k] = bo; S.bl[k] = bl;
      S.J[0][k] = nx;
      S.M[k] = k == 0;
    }
    __syncwarp();
    // Every field takes at least two bytes, so the chain has at most kXrWin / 2 members in the window: after the round of d,
    // members 0 .. 2d-1 are marked, and the rounds up to d = kXrWin / 4 mark them all.  Each round loads everything it needs
    // before it stores (a mark stored early only marks further chain members).
    uint32_t cur = 0;
#pragma unroll 1
    for (uint32_t d = 1; d < kXrWin / 2; d <<= 1, cur ^= 1) {
      int32_t t[8], tt[8];
      uint8_t m[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) t[j] = S.J[cur][32 * j + lane];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const bool in = t[j] >= 0 && (uint32_t)t[j] < L;
        m[j] = in ? S.M[32 * j + lane] : 0;
        tt[j] = in ? S.J[cur][t[j]] : t[j];
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if (m[j]) S.M[t[j]] = 1;
        S.J[cur ^ 1][32 * j + lane] = tt[j];
      }
      __syncwarp();
    }
#pragma unroll 1
    for (int j = 0; j < 8; ++j) {                          // the chain's entries, in wire order, and its last member
      const uint32_t k = 32 * j + lane;
      const int32_t nx = S.nx[k];
      const bool on = k < L && S.M[k];
      if (on && (nx < 0 || (uint32_t)nx >= L)) { S.exit_k = (int32_t)k; S.exit_t = nx; }
      const bool f = on && nx >= 0 && S.bl[k] != ~0u;
      const uint32_t m = __ballot_sync(0xFFFFFFFFu, f);
      const uint32_t i = base + count + __popc(m & ((1u << lane) - 1));
      if (f && slot && i < cap) slot[i] = b200tfs_label_ref{S.bo[k], S.bl[k]};
      count += __popc(m);
    }
    __syncwarp();
    const int32_t ek = S.exit_k, et = S.exit_t;
    __syncwarp();
    if (et == kXrErr) { *err = B200TFS_E_PARSE; return count; }
    if (et == kXrGroup) {                                  // a group: lane 0's cursor skips it
      uint32_t ns = 0;
      if (lane == 0) {
        const uint32_t p0 = c.p, e0 = c.end;
        c.p = s + (uint32_t)ek; c.end = hi;
        const uint32_t t = rd_tag(c);
        if (!c.err) skip_field(c, t);
        ns = c.err ? 0 : c.p;
        c.err = 0; c.p = p0; c.end = e0;
      }
      ns = __shfl_sync(0xFFFFFFFFu, ns, 0);
      if (!ns) { *err = B200TFS_E_PARSE; return count; }
      s = ns;
    } else {
      s += (uint32_t)et;
    }
  }
  return count;
}

__global__ void __launch_bounds__(32 * kXrIndexWarps) xr_index_kernel(const __grid_constant__ XrTables T) {
  __shared__ __align__(16) uint8_t lines[kXrIndexWarps][256];
  __shared__ __align__(16) XrWarpSmem win[kXrIndexWarps];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31, r = blockIdx.x * kXrIndexWarps + warp;
  if (r >= T.n) return;
  const uint8_t* rec = T.w + T.rec_off[r];
  const uint32_t len = (uint32_t)T.rec_len[r];
  for (uint32_t q = 128 * lane; q < len; q += 32 * 128) xr_prefetch_l2(rec + q);
  // lane 0 walks the top level (model_spec, unknown fields); the whole warp finds the entries of every result body
  Cursor c;
  b200tfs_model_spec spec;
  if (lane == 0) { cur_open(c, rec, len, lines[warp]); spec_reset(spec); }
  b200tfs_label_ref* slot = T.ent + T.ent0[r];
  const uint32_t cap = (uint32_t)xr_row_bound(len);
  uint32_t count = 0;
  int err = 0;
#pragma unroll 1
  for (;;) {
    uint32_t lo = 0, hi = 0, more = 0;
    if (lane == 0) { more = xr_next_result(c, spec, &lo, &hi); err = c.err; }
    more = __shfl_sync(0xFFFFFFFFu, more, 0); lo = __shfl_sync(0xFFFFFFFFu, lo, 0); hi = __shfl_sync(0xFFFFFFFFu, hi, 0);
    err = __shfl_sync(0xFFFFFFFFu, err, 0);
    if (!more || err) break;
    count += xr_warp_entries(win[warp], c, rec, len, lo, hi, slot, count, cap, &err);
    if (err) break;
  }
  uint32_t k0 = 0;
  if (!err && T.kind == B200TFS_RESP_CLASSIFY && count) {   // the first example's classes: C, if this is the batch's first
    __syncwarp();
    const b200tfs_label_ref e = slot[0];
    int e2;
    k0 = xr_warp_entries(win[warp], c, rec, len, e.off, e.off + e.len, nullptr, 0, 0, &e2);   // a malformed one: emit reports it
  }
  if (lane) return;
  T.rows[r] = err ? 0 : count;
  T.cls0[r] = k0;
  T.status[r] = err ? B200TFS_E_PARSE : B200TFS_OK;
  T.specs[r] = spec;
}

__global__ void __launch_bounds__(kConcatPlanThreads) xr_scan_kernel(const __grid_constant__ XrTables T) {
  __shared__ unsigned long long warp_sum[kConcatPlanThreads / 32];
  __shared__ unsigned int first;
  if (threadIdx.x == 0) first = ~0u;
  __syncthreads();
  for (uint32_t r = threadIdx.x; r < T.n; r += kConcatPlanThreads) if (T.rows[r]) atomicMin(&first, r);
  __syncthreads();
  const bool cls = T.kind == B200TFS_RESP_CLASSIFY;
  const uint64_t C = cls && first != ~0u ? T.cls0[first] : 0, per = cls ? C : 1;
  uint64_t carry = 0;
  for (uint32_t r0 = 0; r0 < T.n; r0 += kConcatPlanThreads) {   // uniform trip count
    const uint32_t r = r0 + threadIdx.x;
    const uint64_t rows = r < T.n ? T.rows[r] : 0;
    const uint64_t at = concat_scan(rows, carry, warp_sum);
    if (r < T.n) {
      T.row0[r] = at;
      const uint64_t end = (at + rows) * per;
      if (rows && T.status[r] == B200TFS_OK && (end > T.values_cap || (cls && end > T.labels_cap))) T.status[r] = B200TFS_E_SIZE;
    }
  }
  if (threadIdx.x == 0) { T.batch[0] = carry; T.batch[1] = C; T.batch[2] = first; T.batch[3] = 1; }
}

// the response row `row` belongs to: the last one whose first row is <= row (an empty response shares its first row with the
// response behind it, so the last of them is the one that has rows)
__device__ __forceinline__ uint32_t xr_response_of(const XrTables& T, uint64_t row) {
  uint32_t lo = 0, hi = T.n - 1;
  while (lo < hi) {
    const uint32_t m = (lo + hi + 1) >> 1;
    if (T.row0[m] <= row) lo = m; else hi = m - 1;
  }
  return lo;
}

__global__ void __launch_bounds__(kXrEmitThreads) xr_emit_kernel(const __grid_constant__ XrTables T) {
  // every thread's line cache (34 KB), 272 bytes apart so that the threads of a warp reading the same line offset spread over
  // eight banks instead of one
  __shared__ __align__(16) uint8_t lines[kXrEmitThreads][272];
  const uint64_t total = T.batch[0], C = T.batch[1];
  uint32_t* values = reinterpret_cast<uint32_t*>(T.values);
  for (uint64_t row = (uint64_t)blockIdx.x * kXrEmitThreads + threadIdx.x; row < total; row += (uint64_t)gridDim.x * kXrEmitThreads) {
    const uint32_t r = xr_response_of(T, row);
    const b200tfs_label_ref e = T.ent[T.ent0[r] + (row - T.row0[r])];
    const uint8_t* rec = T.w + T.rec_off[r];
    Cursor c;
    if (T.kind == B200TFS_RESP_REGRESS) {
      const uint8_t* p = rec + e.off;
      uint32_t v = 0;
      if (e.len == 5 && p[0] == 0x0D) {       // what a server writes: the value field alone
        v = quiet_f32((uint32_t)p[1] | ((uint32_t)p[2] << 8) | ((uint32_t)p[3] << 16) | ((uint32_t)p[4] << 24));
      } else if (e.len) {
        cur_open(c, p, e.len, lines[threadIdx.x]);
        v = xr_regression(c);
        if (c.err) { atomicMin(&T.status[r], B200TFS_E_PARSE); continue; }
      }
      if (row < T.values_cap) values[row] = v;
    } else {
      cur_open(c, rec, (uint32_t)T.rec_len[r], lines[threadIdx.x]);
      c.p = e.off; c.end = e.off + e.len;
      XrClassSink s{values, T.labels, row * C, C, T.values_cap, T.labels_cap};
      const uint32_t k = xr_classes(c, s);
      if (c.err) atomicMin(&T.status[r], B200TFS_E_PARSE);
      else if (k != C) atomicMin(&T.status[r], B200TFS_E_SHAPE);
    }
  }
}

constexpr uint32_t kXrCompareThreads = 256;
__global__ void __launch_bounds__(kXrCompareThreads) xr_compare_kernel(const __grid_constant__ XrTables T) {
  const uint64_t total = T.batch[0], C = T.batch[1];
  const uint32_t f = (uint32_t)T.batch[2], lane = threadIdx.x & 31;
  constexpr uint32_t kWarps = kXrCompareThreads / 32;
  if (!C || T.status[f] != B200TFS_OK) return;      // no labels, or the batch does not decode anyway
  const uint8_t* first = T.w + T.rec_off[f];
  for (uint64_t row = 1 + (uint64_t)blockIdx.x * kWarps + (threadIdx.x >> 5); row < total; row += (uint64_t)gridDim.x * kWarps) {
    if (!*reinterpret_cast<volatile unsigned long long*>(&T.batch[3])) return;
    const uint32_t r = xr_response_of(T, row);
    if (T.status[r] != B200TFS_OK) continue;        // its labels were not all stored
    const uint8_t* rec = T.w + T.rec_off[r];
    for (uint64_t k = lane; k < C; k += 32) {
      const b200tfs_label_ref a = T.labels[row * C + k], b = T.labels[k];
      bool eq = a.len == b.len;
      for (uint32_t j = 0; eq && j < a.len; ++j) eq = rec[a.off + j] == first[b.off + j];
      if (!eq) { atomicAnd(&T.batch[3], 0ull); break; }
    }
  }
}

__global__ void __launch_bounds__(256) xr_publish_kernel(const __grid_constant__ XrTables T) {
  __shared__ unsigned int bad;
  if (threadIdx.x == 0) bad = ~0u;
  __syncthreads();
  for (uint32_t r = threadIdx.x; r < T.n; r += blockDim.x) {
    const int32_t st = T.status[r];
    T.per_rec_host[3ull * r] = (int64_t)T.row0[r];
    T.per_rec_host[3ull * r + 1] = T.rows[r];
    T.per_rec_host[3ull * r + 2] = st;
    T.specs_host[r] = T.specs[r];
    if (st != B200TFS_OK) atomicMin(&bad, r);
  }
  __syncthreads();
  if (threadIdx.x) return;
  const bool cls = T.kind == B200TFS_RESP_CLASSIFY;
  T.batch_host[0] = (int64_t)T.batch[0];
  T.batch_host[1] = cls ? (int64_t)T.batch[1] : 0;
  T.batch_host[2] = cls ? (int64_t)T.batch[3] : 0;
  T.batch_host[3] = bad == ~0u ? B200TFS_OK : T.status[bad];
  T.batch_host[4] = bad == ~0u ? -1 : (int64_t)bad;
}

cudaError_t launch_example_responses(const XrTables& T, uint32_t emit_ctas, cudaStream_t stream, uint32_t* launched) {
  *launched = 0;
  if (!T.n) return cudaSuccess;
  xr_index_kernel<<<(T.n + kXrIndexWarps - 1) / kXrIndexWarps, 32 * kXrIndexWarps, 0, stream>>>(T);
  xr_scan_kernel<<<1, kConcatPlanThreads, 0, stream>>>(T);
  xr_emit_kernel<<<emit_ctas, kXrEmitThreads, 0, stream>>>(T);
  *launched = 4;
  if (T.kind == B200TFS_RESP_CLASSIFY) { xr_compare_kernel<<<emit_ctas, kXrCompareThreads, 0, stream>>>(T); *launched += 1; }
  xr_publish_kernel<<<1, 256, 0, stream>>>(T);
  return cudaGetLastError();
}
