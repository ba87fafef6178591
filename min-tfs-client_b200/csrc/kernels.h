// kernels.h - launchers exported by kernels.cu to the host side of the library.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/b200tfs.h"
#include "plan.h"
#include "unpad.h"

namespace b200tfs {

// Launch the pack/unpack engine.  plan_dev == nullptr: the plan image (plan_bytes <= kInlinePlanBytes)
// travels in the kernel parameters; otherwise it has already been copied to plan_dev on `stream`.
cudaError_t launch_move(const uint8_t* plan_dev, const uint8_t* plan_host, uint32_t plan_bytes, uint32_t n_tiles,
                        uint32_t n_small, cudaStream_t stream);

// the same engine over a device-resident plan whose items are stored only where PlanHeader::guard says so (codec_host.cpp: the
// narrowing batch decode)
cudaError_t launch_move_guarded(const uint8_t* plan_dev, uint32_t n_tiles, cudaStream_t stream);

// spill: n * spill_per_rec entries of kSpillEntryBytes (walker.h SpillEntry) for dims / value runs beyond the table's inline
// arrays; spill_used[r] receives how many entries record r wanted (more than spill_per_rec: its status is B200TFS_E_SPILL)
constexpr uint32_t kSpillEntryBytes = 32;
cudaError_t launch_parse_responses(const uint8_t* w, const uint64_t* rec_off, const uint64_t* rec_len, int n, int max_outputs,
                                   b200tfs_output* outs, int32_t* n_outs, b200tfs_model_spec* specs, int32_t* status,
                                   void* spill, uint32_t spill_per_rec, uint32_t* spill_used, cudaStream_t stream);
cudaError_t launch_parse_tensors(const uint8_t* w, const uint64_t* rec_off, const uint64_t* rec_len, int n, b200tfs_output* outs,
                                 int32_t* status, void* spill, uint32_t spill_per_rec, uint32_t* spill_used, cudaStream_t stream);

cudaError_t launch_decode_fused(const FusedParams& fp, uint32_t grid, cudaStream_t stream);
constexpr uint32_t kStageVecsHost = 2048;   // == kStageVecs (kernels.cu): launches with fatter tiles run the TMA-staged batch kernel
uint32_t tiles_for_host(uint64_t n_out, uint32_t vpt);
// pad elements [have, n_elems) of dst with element have-1 (zeros if have == 0); have from the host or, if have_dev, the device
cudaError_t launch_fill_edge(uint8_t* dst, uint32_t elem_size, uint64_t have, const unsigned long long* have_dev, uint64_t n_elems,
                             cudaStream_t stream);
// packed varints (varint_kernels.cuh): the tables and counters every kernel uses are addressed through VarTables
cudaError_t launch_frame_requests(const FrameTables& ft, cudaStream_t stream);
cudaError_t launch_venc_len(const VarTables& tb, cudaStream_t stream);
cudaError_t launch_venc_emit(const VarTables& tb, cudaStream_t stream);
cudaError_t launch_vdec_count(const VarTables& tb, cudaStream_t stream);
cudaError_t launch_vdec_emit(const VarTables& tb, cudaStream_t stream);
// packed-varint outputs of the single-launch decode: the plan kernel, then count + emit over the tables it built (tb.n_tiles is
// the host's bound, tb.n_tiles_dev the real count; each kernel runs at most max_ctas CTAs and strides over the tiles)
cudaError_t launch_vdec_plan(const VarPlan& vp, cudaStream_t stream);
// (pm: the padded decode's emit, every element at its padded position)
cudaError_t launch_vdec_dev(const VarTables& tb, uint32_t max_ctas, cudaStream_t stream, const VarPadMap* pm = nullptr);
// b200tfs_decode_concat: concat_plan_kernel, then move_kernel over the plan image it wrote, with move_grid CTAs (the host's bound
// on the tiles; the CTAs past the plan's own count leave at once)
// (strings: concat_plan_strings_kernel, which places the DT_STRING outputs' offsets too)
cudaError_t launch_concat_plan(const ConcatPlan& cp, uint32_t move_grid, cudaStream_t stream, bool strings = false);
// b200tfs_decode_concat_strings, behind launch_concat_plan: index, scan, copy and fix (string_kernels.cuh); the index runs a warp
// per (record, key), copy and fix run grid CTAs striding over the chunks
cudaError_t launch_concat_strings(const StrTables& T, uint32_t grid, cudaStream_t stream);
// b200tfs_decode_padded: padded_plan_kernel, then padded_emit_kernel with emit_grid CTAs striding over the chunks
// (strings: padded_plan_strings_kernel, which places the DT_STRING outputs' offsets too)
cudaError_t launch_padded(const PaddedPlan& pp, uint32_t emit_grid, cudaStream_t stream, bool strings = false);
// b200tfs_decode_padded_strings, behind launch_padded: index, scan, copy and fix (padded_kernels.cuh); the index runs a warp per
// (record, key), copy and fix run grid CTAs striding over the positions
cudaError_t launch_padded_strings(const PadStrTables& T, uint32_t grid, cudaStream_t stream);
// tf.Example requests (example_kernels.cuh): count + scan (when T.n_tiles), emit, frame; *launched receives how many kernels.
// ctx (device, one ExCtxRef per request; NULL: a call without contexts) selects the frame kernel that writes the contexts.
// lists (NULL: a call without PREDICT_ELWCS requests): the frame runs before the emits, and the list emits after the others.
// dev (NULL: no PREDICT_ELWCS request with device list sizes): the frame also plans those requests' spans, emitted by one more kernel.
cudaError_t launch_example_requests(const ExTables& T, int mode, cudaStream_t stream, uint32_t* launched, const ExCtxRef* ctx,
                                    uint32_t n_seq_tiles, uint32_t n_seq_spans, const ExLists* lists = nullptr,
                                    const ExDevLists* dev = nullptr);
// Classify / Regress responses (example_resp_kernels.cuh): index, scan, emit, [label compare,] publish; emit_ctas CTAs stride over
// the rows; *launched receives how many kernels
cudaError_t launch_example_responses(const XrTables& T, uint32_t emit_ctas, cudaStream_t stream, uint32_t* launched);
// MultiInference responses (multi_resp_kernels.cuh): index, then scan, emit, [label compare,] publish on each of the M.n_tasks
// views (host array); *launched receives how many kernels
cudaError_t launch_multi_inference_responses(const MiTables& M, const XrTables* views, uint32_t emit_ctas, cudaStream_t stream,
                                             uint32_t* launched);
// PredictRequests cut out of padded tensors (unpad_kernels.cuh): plan, [varint count,] layout, frame, move over move_grid CTAs (the
// host's bound on the tiles), [varint emit]; *launched receives how many kernels
cudaError_t launch_unpad(const UnpadPlan& up, uint32_t move_grid, cudaStream_t stream, uint32_t* launched);

}  // namespace b200tfs
