// multi_resp_kernels.cuh - MultiInference responses: a batch of responses into one value / score array per task (plan.h MiTables;
// planned by example_host.inc; the walk is multi_walk.h).  Included by kernels.cu inside namespace b200tfs, after
// example_resp_kernels.cuh, whose kernels decode each task.
//
//   mi_index_kernel    one warp per response: lane 0 walks `results` and each result's fields (mi_result_case) and parses the
//                      entries of every result no task decodes to the end (mi_check_run), the whole warp
//                      finds the entries of the surviving member's bodies (xr_warp_entries) and writes them into the response's
//                      slots, task after task; per (response, task) it fills the task's ent0, rows, cls0, specs and status
//   then, per task, on the task's XrTables view: xr_scan_kernel, xr_emit_kernel, [xr_compare_kernel,] xr_publish_kernel
//
// What the reference does here: MultiInferenceResponse.FromString and a Python loop over each result's entries.

__global__ void __launch_bounds__(32 * kXrIndexWarps) mi_index_kernel(const __grid_constant__ MiTables M) {
  __shared__ __align__(16) uint8_t lines[kXrIndexWarps][256];
  __shared__ __align__(16) XrWarpSmem win[kXrIndexWarps];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31, r = blockIdx.x * kXrIndexWarps + warp;
  if (r >= M.n) return;
  const uint8_t* rec = M.w + M.rec_off[r];
  const uint32_t len = (uint32_t)M.rec_len[r];
  for (uint32_t q = 128 * lane; q < len; q += 32 * 128) xr_prefetch_l2(rec + q);
  Cursor c;
  if (lane == 0) cur_open(c, rec, len, lines[warp]);
  const uint64_t e0 = M.E0[r];
  b200tfs_label_ref* slot = M.ent + e0;
  const uint32_t cap = (uint32_t)xr_row_bound(len);
  uint32_t count = 0, k = 0;
  int err = 0;
#pragma unroll 1
  for (;; ++k) {
    // lane 0: the next result, and (for a task's result) its model_spec, surviving member and where that member's run starts
    uint32_t more = 0, rhi = 0, kase = 0, from = 0;
    b200tfs_model_spec spec;
    if (lane == 0) {
      uint32_t rlo;
      more = mi_next_result(c, &rlo, &rhi);
      if (more) {
        spec_reset(spec);
        mi_result_case(c, rlo, rhi, spec, &kase, &from);
        // a result no task decodes - past the tasks, or another member than its task's -: its entries are only checked
        if (k >= M.n_tasks || kase != mi_case_of(M.kinds[k])) mi_check_run(c, kase, from, rhi);
      }
      err = c.err;
    }
    more = __shfl_sync(0xFFFFFFFFu, more, 0); err = __shfl_sync(0xFFFFFFFFu, err, 0);
    if (!more || err) break;
    if (k >= M.n_tasks) continue;    // a result past the tasks: checked and counted only (the response is B200TFS_E_SHAPE)
    kase = __shfl_sync(0xFFFFFFFFu, kase, 0); from = __shfl_sync(0xFFFFFFFFu, from, 0); rhi = __shfl_sync(0xFFFFFFFFu, rhi, 0);
    const uint32_t base = count;
    const bool match = kase == mi_case_of(M.kinds[k]);
    if (match) {                      // the entries of every occurrence of the member from `from` on
      uint32_t p = from;
#pragma unroll 1
      for (;;) {
        uint32_t blo = 0, bhi = 0, got = 0;
        if (lane == 0) {
          const uint32_t p0 = c.p, e0c = c.end;
          c.p = p; c.end = rhi;
          got = mi_next_member(c, kase, &blo, &bhi);
          p = c.p;
          c.p = p0; c.end = e0c;
        }
        got = __shfl_sync(0xFFFFFFFFu, got, 0);
        if (!got) break;
        blo = __shfl_sync(0xFFFFFFFFu, blo, 0); bhi = __shfl_sync(0xFFFFFFFFu, bhi, 0);
        count += xr_warp_entries(win[warp], c, rec, len, blo, bhi, slot, count, cap, &err);
        if (err) break;
      }
      if (err) break;
    }
    const uint32_t rows = count - base;
    uint32_t k0 = 0;
    if (match && M.kinds[k] == B200TFS_RESP_CLASSIFY && rows) {   // the first example's classes: C, if this is the task's first
      __syncwarp();
      const b200tfs_label_ref e = slot[base];
      int e2;
      k0 = xr_warp_entries(win[warp], c, rec, len, e.off, e.off + e.len, nullptr, 0, 0, &e2);   // a malformed one: emit reports it
    }
    if (lane == 0) {
      const uint64_t i = (uint64_t)k * M.n + r;
      M.ent0[i] = e0 + base;
      M.rows[i] = match ? rows : 0;
      M.cls0[i] = k0;
      M.status[i] = match ? B200TFS_OK : B200TFS_E_SHAPE;
      M.specs[i] = spec;
    }
  }
  if (lane || (!err && k == M.n_tasks)) return;
  // a malformed response (every task B200TFS_E_PARSE, no rows), or one with another result count (every task B200TFS_E_SHAPE;
  // the tasks without a result have no rows)
  for (uint32_t t = 0; t < M.n_tasks; ++t) {
    const uint64_t i = (uint64_t)t * M.n + r;
    if (err || t >= k) {
      M.ent0[i] = e0; M.rows[i] = 0; M.cls0[i] = 0;
      spec_reset(M.specs[i]);
    }
    M.status[i] = err ? B200TFS_E_PARSE : B200TFS_E_SHAPE;
  }
}

cudaError_t launch_multi_inference_responses(const MiTables& M, const XrTables* views, uint32_t emit_ctas, cudaStream_t stream,
                                             uint32_t* launched) {
  *launched = 0;
  if (!M.n) return cudaSuccess;
  mi_index_kernel<<<(M.n + kXrIndexWarps - 1) / kXrIndexWarps, 32 * kXrIndexWarps, 0, stream>>>(M);
  *launched = 1;
  for (uint32_t t = 0; t < M.n_tasks; ++t) {
    const XrTables& T = views[t];
    xr_scan_kernel<<<1, kConcatPlanThreads, 0, stream>>>(T);
    xr_emit_kernel<<<emit_ctas, kXrEmitThreads, 0, stream>>>(T);
    *launched += 3;
    if (T.kind == B200TFS_RESP_CLASSIFY) { xr_compare_kernel<<<emit_ctas, kXrCompareThreads, 0, stream>>>(T); *launched += 1; }
    xr_publish_kernel<<<1, 256, 0, stream>>>(T);
  }
  return cudaGetLastError();
}
