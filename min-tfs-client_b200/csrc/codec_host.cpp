// codec_host.cpp - host half of libb200tfs.so: the C ABI of include/b200tfs.h, the wire-size
// arithmetic, the header planner (tags, varint lengths, dims, keys - everything on the wire that is
// not tensor payload) and the launch plans handed to the kernels in kernels.cu.
//
// The planner restates the framing the reference gets from protobuf for
//   TensorProto{dtype, tensor_shape{dim{size}}, <typed packed field>}      tensors.py:28-35
//   PredictRequest{model_spec{name, version{value}}, inputs{key -> proto}}  requests.py:41-48
// (proto3 rules: fields in ascending number, zero scalars elided, packed repeated scalars, map entries
// always carry key and value) - SURVEY.md 8(a) a1-a3 and quirks Q1-Q5.  There is deliberately no CPU
// implementation of the payload path here: payload bytes only ever move inside the CUDA kernels.
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/b200tfs.h"
#include "example_walk.h"
#include "framing.h"
#include "kernels.h"
#include "plan.h"
#include "string_walk.h"
#include "tpl.h"
#include "walker.h"
#include "wire.h"

using namespace b200tfs;

// ------------------------------------------------------------------------------------------------
// errors
// ------------------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";

static int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof g_err, fmt, ap);
  va_end(ap);
  return code;
}

#define CU(call)                                                                                   \
  do {                                                                                             \
    cudaError_t e_ = (call);                                                                       \
    if (e_ != cudaSuccess) return fail(B200TFS_E_CUDA, "%s: %s", #call, cudaGetErrorString(e_));   \
  } while (0)

// ------------------------------------------------------------------------------------------------
// context
// ------------------------------------------------------------------------------------------------
namespace {

struct Growable {  // device or pinned buffer that only grows
  void* p = nullptr;
  uint64_t cap = 0;
};

constexpr int kSlots = 4;

struct Slot {  // one in-flight plan upload: pinned image + device image + completion event
  Growable host, dev;
  cudaEvent_t done = nullptr;
  bool pending = false;
};

}  // namespace

struct MeasuredTensor {     // what b200tfs_measure learnt about one varint tensor (device addresses of its counters)
  uint64_t n_elems = 0, packed_len = 0;
  int32_t dtype = 0;
  void* tile_val = nullptr;
  void* group_sum = nullptr;
  void* total = nullptr;
};

struct b200tfs_ctx {
  int device = 0;
  int sm_count = 132;   // H100 SXM; replaced by the device's own count when the context is created
  cudaStream_t stream = nullptr;       // the stream every call is ordered on: the context's own, or the caller's (b200tfs_set_stream)
  cudaStream_t own_stream = nullptr;
  cudaStream_t aux_stream = nullptr;   // uploads done at capture time, outside the graph being recorded; the pipelined host path's H2D copies
  cudaStream_t d2h_stream = nullptr;   // the pipelined host path's D2H copies
  static constexpr int kPipeMax = 8;   // slices of one pipelined host call
  cudaEvent_t pipe_ev[2 * kPipeMax + 2] = {};
  uint64_t pipe_min = 1ull << 20;      // *_host calls moving at least this many payload bytes are sliced (B200TFS_PIPELINE_MIN; 0 = never)
  int pipe_max = 4;                    // at most this many slices (B200TFS_PIPELINE_SLICES, 2..kPipeMax): every slice costs ~7 driver calls
  uint64_t pipelined_calls = 0;        // how many host calls took the sliced path (tests)
  uint64_t direct_calls = 0;           // ... and how many wrote their output straight into the caller's pinned buffer
  bool opt_direct_out = true;          // B200TFS_DIRECT_OUT=0: always stage the output on the device and copy it back
  Growable guard_dev;                  // the narrowing batch decode's per-record verdicts (FusedParams::guard)
  uint32_t decode_cast = 0;            // b200tfs_set_decode_cast: DT_FLOAT outputs of the single-launch decode leave as DT_HALF / DT_BFLOAT16
  uint32_t decode_varints = 0;         // b200tfs_set_decode_varints: the single-launch decode decodes packed-varint outputs too
  bool fused_varints = false;          // ... and the last one did: b200tfs_decode_results folds the statuses vdec_plan_kernel's jobs left
  Growable vdec_dev;                   // its device-built tables and counters (VarPlan)
  Slot slots[kSlots];
  int next_slot = 0;
  Growable scratch_dev;   // parse tables / varint tile tables
  Growable scratch_host;  // pinned mirror of the parse tables
  Growable stage_dev;     // *_host entry points: tensors (encode) or wire (decode) staged on the device
  Growable arena_dev;     // *_host entry points: wire arena (encode) / unpacked tensors (decode)
  uint64_t launches = 0;
  uint32_t tile_bytes_override = 0;
  bool capturing = false;   // between b200tfs_capture_begin / _end: no syncs; uploads get buffers that live as long as the context
  std::vector<Slot*> graph_slots;  // plan images referenced by captured graphs
  Growable fused_host;      // decode_fused tables: pinned host memory the kernel writes directly
  void* tpl_dev = nullptr;  // two framing templates (device), used alternately by successive decode launches
  uint32_t tpl_flip = 0;
  TplInline* tpl_pinned = nullptr;   // where a kernel that learns a template leaves its inline part (pinned, mapped)
  TplInline tpl_known{};             // the newest template the host knows: its own walk of a host-resident record 0, or tpl_pinned
                                     // as found with the stream idle; rides in the kernel parameters of the next single-response launch
  uint32_t serial = 0;               // stamp of the next template learnt
  cudaEvent_t tpl_event = nullptr;   // recorded behind every eager decode launch: once it has completed, tpl_pinned is current
  bool tpl_event_pending = false;
  bool opt_no_inline = false;        // B200TFS_NO_INLINE_TEMPLATE=1: never hand the template over in the kernel parameters (experiments)
  uint64_t stage_shift = 0;          // *_host decode: the wire sits at stage_dev + stage_shift (placed so that the payload is 16-byte aligned)
  int32_t fused_n = 0;      // records of the last b200tfs_decode_responses
  std::vector<int32_t> pending_status;   // varint decode: which output each status word in scratch_host belongs to
  // counters left by b200tfs_measure, keyed by tensor address; consumed by the encode that follows
  Growable measured_dev;
  uint64_t measured_used = 0;
  std::unordered_map<const void*, MeasuredTensor> measured;
  // spill area of the two-phase parse: dims / value runs beyond the table's inline arrays (walker.h SpillEntry)
  Growable spill_dev;
  std::vector<SpillEntry> spill_host;   // host copy of the last parse's area (empty when no record spilled)
  uint32_t spill_per_rec = 16;          // entries per record the next parse starts with
  uint32_t spill_last_per = 0;          // geometry of spill_host
  int32_t spill_last_n = 0;
  Growable gather_dev;                  // unpack: strided / many-run varint outputs are first gathered into one stream here
  Growable enc_host;                    // b200tfs_encode_requests_async: rec_off | rec_len | status, written by frame_requests_kernel (pinned)
  int32_t enc_n = 0;
  bool has_graphs = false;              // a CUDA graph captured on this context refers to the scratch buffers: they may not move any more
  // the per-key decodes' most recent call, what their results calls answer for: records, keys, destinations and where the
  // table, the varint statuses, the specs and the record statuses lie in the scratch buffer
  struct KeyResults {
    int32_t n = 0, k = 0;
    uint8_t* dst[B200TFS_CONCAT_MAX_KEYS] = {};
    uint64_t vouts = 0, vstat = 0, specs = 0, status = 0;
  };
  Growable concat_dev;                  // b200tfs_decode_concat: parse table, varint tables, plan image (KeyLayout)
  KeyResults concat_res;
  Growable padded_dev;                  // b200tfs_decode_padded: parse table, varint tables, descriptors (KeyLayout)
  KeyResults padded_res;
  Growable xr_dev;                      // b200tfs_decode_example_responses: entry slots and per-response tables (XrLayout)
  Growable xr_host;                     // ... and the results its publish kernel leaves in pinned memory (XrResultsLayout)
  int32_t xr_n = 0;                     // responses of its most recent call, what b200tfs_example_response_results answers for
  Growable mi_dev, mi_host;             // b200tfs_decode_multi_inference_responses: the same, for every task (MiLayout)
  int32_t mi_n = 0, mi_tasks = 0;       // responses and tasks of its most recent call
  Growable unpad_dev;                   // b200tfs_encode_padded_requests_async: boxes, varint jobs and counters, move plan (UnpadLayout)
};

// `baked`: the buffer's address ends up inside captured graphs (every context-owned scratch buffer except the plan-upload
// slots, which captured launches replace by private ones).  Once a graph exists, such a buffer must not be reallocated:
// replays would write through the stale address.  Size everything with the largest call BEFORE capturing.
static const char* kGraphPinned = "a CUDA graph captured on this context refers to its scratch buffers, which this larger call would have to "
                                  "reallocate: run the largest call once before capturing, or use another context";
static int grow_dev(b200tfs_ctx* c, Growable& g, uint64_t need, bool baked = true) {
  if (need <= g.cap) return B200TFS_OK;
  if (c->capturing) return fail(B200TFS_E_ARG, "scratch buffer would have to grow during graph capture: run the call once before capturing");
  if (baked && c->has_graphs) return fail(B200TFS_E_ARG, "%s", kGraphPinned);
  uint64_t cap = std::max<uint64_t>(need, g.cap * 2);
  cap = (cap + 0xFFFFull) & ~0xFFFFull;
  CU(cudaStreamSynchronize(c->stream));
  if (g.p) CU(cudaFree(g.p));
  g.p = nullptr; g.cap = 0;
  CU(cudaMalloc(&g.p, cap));
  g.cap = cap;
  return B200TFS_OK;
}
static int grow_host(b200tfs_ctx* c, Growable& g, uint64_t need, bool baked = true) {
  if (need <= g.cap) return B200TFS_OK;
  if (c->capturing) return fail(B200TFS_E_ARG, "scratch buffer would have to grow during graph capture: run the call once before capturing");
  if (baked && c->has_graphs) return fail(B200TFS_E_ARG, "%s", kGraphPinned);
  uint64_t cap = std::max<uint64_t>(need, g.cap * 2);
  cap = (cap + 0xFFFull) & ~0xFFFull;
  CU(cudaStreamSynchronize(c->stream));
  if (g.p) CU(cudaFreeHost(g.p));
  g.p = nullptr; g.cap = 0;
  CU(cudaHostAlloc(&g.p, cap, cudaHostAllocPortable | cudaHostAllocMapped));
  g.cap = cap;
  return B200TFS_OK;
}

// claim an upload slot with room for `bytes` in both images
static int claim_slot(b200tfs_ctx* c, uint64_t bytes, Slot** out) {
  if (c->capturing) {
    // a captured launch must keep its plan image for as long as the graph may be replayed: give it private
    // buffers (the upload itself is recorded as a copy node and simply repeats on every replay)
    Slot* g = new Slot();
    cudaError_t e = cudaHostAlloc(&g->host.p, bytes, cudaHostAllocPortable);
    if (e == cudaSuccess) e = cudaMalloc(&g->dev.p, bytes);
    if (e != cudaSuccess) {
      if (g->host.p) cudaFreeHost(g->host.p);
      delete g;
      return fail(B200TFS_E_CUDA, "plan buffers for a captured launch: %s", cudaGetErrorString(e));
    }
    g->host.cap = g->dev.cap = bytes;
    c->graph_slots.push_back(g);
    *out = g;
    return B200TFS_OK;
  }
  Slot& s = c->slots[c->next_slot];
  c->next_slot = (c->next_slot + 1) % kSlots;
  if (s.pending) { CU(cudaEventSynchronize(s.done)); s.pending = false; }
  int rc;
  if ((rc = grow_host(c, s.host, bytes, false))) return rc;
  if ((rc = grow_dev(c, s.dev, bytes, false))) return rc;
  *out = &s;
  return B200TFS_OK;
}

// Bring a slot's pinned image to its device image.  While a graph is being captured the slot is private to that graph and its
// image never changes (plans, tables and framing programs are functions of the call's arguments, which a graph freezes
// anyway): it is copied NOW, on a side stream, instead of being recorded as a copy node that every replay would repeat
// (each such node costs stream time on every replay; a captured C3 encode had three of them).
static int upload_slot(b200tfs_ctx* c, Slot* slot, uint64_t bytes) {
  if (c->capturing) {
    CU(cudaMemcpyAsync(slot->dev.p, slot->host.p, bytes, cudaMemcpyHostToDevice, c->aux_stream));
    CU(cudaStreamSynchronize(c->aux_stream));
    return B200TFS_OK;
  }
  CU(cudaMemcpyAsync(slot->dev.p, slot->host.p, bytes, cudaMemcpyHostToDevice, c->stream));
  if (slot->done) { CU(cudaEventRecord(slot->done, c->stream)); slot->pending = true; }
  return B200TFS_OK;
}

// The regions of a scratch buffer or an upload image, laid out one behind the other: take() hands out a region's offset,
// `end` is where the last one ends.  Each layout is one function that the code sizing the buffer and the code using it both call.
struct Layout {
  uint64_t end = 0;
  uint64_t take(uint64_t bytes, uint64_t align = 16) {
    const uint64_t at = (end + align - 1) & ~(align - 1);
    end = at + bytes;
    return at;
  }
};

// One host array of an upload image, and where it goes
struct ImagePart { uint64_t off; const void* src; uint64_t bytes; };
struct NoFill { void operator()(uint8_t*, uint8_t*) const {} };

// Claim an upload slot for an image of `bytes`, copy every part to its offset, let `fill(host, dev)` write what depends on the
// device address, and bring the first `sent` bytes (all of them by default) to the device.  *dev receives the device base.
template <class Fill = NoFill>
static int upload_image(b200tfs_ctx* c, uint64_t bytes, std::initializer_list<ImagePart> parts, uint8_t** dev, Slot** out = nullptr,
                        Fill&& fill = Fill(), uint64_t sent = ~0ull) {
  Slot* slot;
  int rc = claim_slot(c, bytes, &slot);
  if (rc) return rc;
  uint8_t* h = (uint8_t*)slot->host.p;
  for (const ImagePart& p : parts) if (p.bytes) memcpy(h + p.off, p.src, p.bytes);
  fill(h, (uint8_t*)slot->dev.p);
  if ((rc = upload_slot(c, slot, std::min(sent, bytes)))) return rc;
  *dev = (uint8_t*)slot->dev.p;
  if (out) *out = slot;
  return B200TFS_OK;
}

extern "C" {

int b200tfs_abi_version(void) { return B200TFS_ABI_VERSION; }
const char* b200tfs_last_error(void) { return g_err; }

int b200tfs_device_count(int* count) {
  if (!count) return fail(B200TFS_E_ARG, "count is NULL");
  *count = 0;
  cudaError_t e = cudaGetDeviceCount(count);
  if (e != cudaSuccess) { *count = 0; return fail(B200TFS_E_CUDA, "cudaGetDeviceCount: %s", cudaGetErrorString(e)); }
  return B200TFS_OK;
}

int b200tfs_create(int device, b200tfs_ctx** out) {
  if (!out) return fail(B200TFS_E_ARG, "out is NULL");
  *out = nullptr;
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0)
    return fail(B200TFS_E_CUDA, "no CUDA device (%s): this library has no CPU path", e == cudaSuccess ? "count=0" : cudaGetErrorString(e));
  if (device < 0 || device >= n) return fail(B200TFS_E_ARG, "device %d out of range (have %d)", device, n);
  CU(cudaSetDevice(device));
  b200tfs_ctx* c = new b200tfs_ctx();
  c->device = device;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) c->sm_count = prop.multiProcessorCount;
  e = cudaStreamCreateWithFlags(&c->own_stream, cudaStreamNonBlocking);
  if (e != cudaSuccess) { delete c; return fail(B200TFS_E_CUDA, "cudaStreamCreate: %s", cudaGetErrorString(e)); }
  c->stream = c->own_stream;
  e = cudaStreamCreateWithFlags(&c->aux_stream, cudaStreamNonBlocking);
  if (e != cudaSuccess) { delete c; return fail(B200TFS_E_CUDA, "cudaStreamCreate: %s", cudaGetErrorString(e)); }
  for (auto& s : c->slots) {
    e = cudaEventCreateWithFlags(&s.done, cudaEventDisableTiming);
    if (e != cudaSuccess) { delete c; return fail(B200TFS_E_CUDA, "cudaEventCreate: %s", cudaGetErrorString(e)); }
  }
  const char* tb = getenv("B200TFS_TILE_BYTES");
  if (tb) c->tile_bytes_override = (uint32_t)strtoul(tb, nullptr, 10);
  const char* oi = getenv("B200TFS_NO_INLINE_TEMPLATE");
  c->opt_no_inline = oi && oi[0] == '1';
  e = cudaEventCreateWithFlags(&c->tpl_event, cudaEventDisableTiming);
  if (e != cudaSuccess) { delete c; return fail(B200TFS_E_CUDA, "cudaEventCreate: %s", cudaGetErrorString(e)); }
  e = cudaStreamCreateWithFlags(&c->d2h_stream, cudaStreamNonBlocking);
  for (auto& ev : c->pipe_ev) if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
  if (e != cudaSuccess) { delete c; return fail(B200TFS_E_CUDA, "pipeline stream / events: %s", cudaGetErrorString(e)); }
  const char* pm = getenv("B200TFS_PIPELINE_MIN");
  if (pm) c->pipe_min = strtoull(pm, nullptr, 10);
  const char* pd = getenv("B200TFS_DIRECT_OUT");
  if (pd && pd[0] == '0') c->opt_direct_out = false;
  const char* ps = getenv("B200TFS_PIPELINE_SLICES");
  if (ps) c->pipe_max = std::min<int>(b200tfs_ctx::kPipeMax, std::max(2, atoi(ps)));
  *out = c;
  return B200TFS_OK;
}

int b200tfs_destroy(b200tfs_ctx* c) {
  if (!c) return B200TFS_OK;
  cudaSetDevice(c->device);
  cudaStreamSynchronize(c->stream);
  if (c->stream != c->own_stream) cudaStreamSynchronize(c->own_stream);
  for (auto& s : c->slots) {
    if (s.host.p) cudaFreeHost(s.host.p);
    if (s.dev.p) cudaFree(s.dev.p);
    if (s.done) cudaEventDestroy(s.done);
  }
  if (c->fused_host.p) cudaFreeHost(c->fused_host.p);
  if (c->tpl_dev) cudaFree(c->tpl_dev);
  if (c->tpl_pinned) cudaFreeHost(c->tpl_pinned);
  if (c->tpl_event) cudaEventDestroy(c->tpl_event);
  for (Slot* g : c->graph_slots) { cudaFreeHost(g->host.p); cudaFree(g->dev.p); delete g; }
  if (c->scratch_dev.p) cudaFree(c->scratch_dev.p);
  if (c->spill_dev.p) cudaFree(c->spill_dev.p);
  if (c->gather_dev.p) cudaFree(c->gather_dev.p);
  if (c->guard_dev.p) cudaFree(c->guard_dev.p);
  if (c->vdec_dev.p) cudaFree(c->vdec_dev.p);
  if (c->concat_dev.p) cudaFree(c->concat_dev.p);
  if (c->padded_dev.p) cudaFree(c->padded_dev.p);
  if (c->xr_dev.p) cudaFree(c->xr_dev.p);
  if (c->unpad_dev.p) cudaFree(c->unpad_dev.p);
  if (c->xr_host.p) cudaFreeHost(c->xr_host.p);
  if (c->mi_dev.p) cudaFree(c->mi_dev.p);
  if (c->mi_host.p) cudaFreeHost(c->mi_host.p);
  if (c->enc_host.p) cudaFreeHost(c->enc_host.p);
  if (c->measured_dev.p) cudaFree(c->measured_dev.p);
  if (c->scratch_host.p) cudaFreeHost(c->scratch_host.p);
  if (c->stage_dev.p) cudaFree(c->stage_dev.p);
  if (c->arena_dev.p) cudaFree(c->arena_dev.p);
  cudaStreamDestroy(c->own_stream);
  if (c->aux_stream) cudaStreamDestroy(c->aux_stream);
  if (c->d2h_stream) cudaStreamDestroy(c->d2h_stream);
  for (auto& ev : c->pipe_ev) if (ev) cudaEventDestroy(ev);
  delete c;
  return B200TFS_OK;
}

int b200tfs_set_stream(b200tfs_ctx* c, void* stream) {
  if (!c) return fail(B200TFS_E_ARG, "ctx is NULL");
  if (c->capturing) return fail(B200TFS_E_ARG, "cannot change streams during graph capture");
  cudaStream_t next = stream ? (cudaStream_t)stream : c->own_stream;
  if (next == c->stream) return B200TFS_OK;
  CU(cudaSetDevice(c->device));
  // work already queued on the old stream (plan uploads, kernels reading the scratch buffers) must be visible to the new one:
  // an event edge, not a host synchronise
  cudaEvent_t e;
  CU(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  cudaError_t rc = cudaEventRecord(e, c->stream);
  if (rc == cudaSuccess) rc = cudaStreamWaitEvent(next, e, 0);
  cudaEventDestroy(e);
  if (rc != cudaSuccess) return fail(B200TFS_E_CUDA, "switching streams: %s", cudaGetErrorString(rc));
  c->stream = next;
  return B200TFS_OK;
}

int b200tfs_sync(b200tfs_ctx* c) {
  if (!c) return fail(B200TFS_E_ARG, "ctx is NULL");
  if (c->capturing) return fail(B200TFS_E_ARG, "cannot synchronise during graph capture");
  CU(cudaStreamSynchronize(c->stream));
  return B200TFS_OK;
}
void* b200tfs_stream(b200tfs_ctx* c) { return c ? (void*)c->stream : nullptr; }
int b200tfs_kernel_launches(b200tfs_ctx* c, uint64_t* count) {
  if (!c || !count) return fail(B200TFS_E_ARG, "NULL argument");
  *count = c->launches;
  return B200TFS_OK;
}

// ---- memory / events ------------------------------------------------------------------------
int b200tfs_malloc(b200tfs_ctx* c, uint64_t bytes, void** dptr) {
  if (!c || !dptr) return fail(B200TFS_E_ARG, "NULL argument");
  CU(cudaSetDevice(c->device));
  CU(cudaMalloc(dptr, bytes ? bytes : 1));
  return B200TFS_OK;
}
int b200tfs_free(b200tfs_ctx* c, void* dptr) {
  if (!c) return fail(B200TFS_E_ARG, "ctx is NULL");
  CU(cudaSetDevice(c->device));
  CU(cudaFree(dptr));
  return B200TFS_OK;
}
int b200tfs_host_alloc(uint64_t bytes, void** hptr) {
  if (!hptr) return fail(B200TFS_E_ARG, "hptr is NULL");
  CU(cudaHostAlloc(hptr, bytes ? bytes : 1, cudaHostAllocPortable));
  return B200TFS_OK;
}
int b200tfs_host_free(void* hptr) { CU(cudaFreeHost(hptr)); return B200TFS_OK; }
int b200tfs_memcpy_h2d(b200tfs_ctx* c, void* d, const void* h, uint64_t n) {
  if (!c) return fail(B200TFS_E_ARG, "ctx is NULL");
  if (n) CU(cudaMemcpyAsync(d, h, n, cudaMemcpyHostToDevice, c->stream));
  return B200TFS_OK;
}
int b200tfs_memcpy_d2h(b200tfs_ctx* c, void* h, const void* d, uint64_t n) {
  if (!c) return fail(B200TFS_E_ARG, "ctx is NULL");
  if (n) CU(cudaMemcpyAsync(h, d, n, cudaMemcpyDeviceToHost, c->stream));
  return B200TFS_OK;
}
int b200tfs_memcpy_d2d(b200tfs_ctx* c, void* d, const void* s, uint64_t n) {
  if (!c) return fail(B200TFS_E_ARG, "ctx is NULL");
  if (n) CU(cudaMemcpyAsync(d, s, n, cudaMemcpyDeviceToDevice, c->stream));
  return B200TFS_OK;
}
int b200tfs_memset(b200tfs_ctx* c, void* d, int v, uint64_t n) {
  if (!c) return fail(B200TFS_E_ARG, "ctx is NULL");
  if (n) CU(cudaMemsetAsync(d, v, n, c->stream));
  return B200TFS_OK;
}
int b200tfs_event_create(void** ev) {
  if (!ev) return fail(B200TFS_E_ARG, "ev is NULL");
  cudaEvent_t e;
  CU(cudaEventCreate(&e));
  *ev = e;
  return B200TFS_OK;
}
int b200tfs_event_destroy(void* ev) { CU(cudaEventDestroy((cudaEvent_t)ev)); return B200TFS_OK; }
int b200tfs_event_record(b200tfs_ctx* c, void* ev) {
  if (!c) return fail(B200TFS_E_ARG, "ctx is NULL");
  CU(cudaEventRecord((cudaEvent_t)ev, c->stream));
  return B200TFS_OK;
}
int b200tfs_event_sync(void* ev) { CU(cudaEventSynchronize((cudaEvent_t)ev)); return B200TFS_OK; }
int b200tfs_event_elapsed_ms(void* a, void* b, float* ms) {
  if (!ms) return fail(B200TFS_E_ARG, "ms is NULL");
  CU(cudaEventElapsedTime(ms, (cudaEvent_t)a, (cudaEvent_t)b));
  return B200TFS_OK;
}

// ---- dtype table -------------------------------------------------------------------------------
int b200tfs_dtype_size(int32_t dt) { return (int)dtype_info(dt).elem_size; }
int b200tfs_dtype_field(int32_t dt) { return (int)dtype_info(dt).field; }
int b200tfs_cast_supported(int32_t src, int32_t wire) {
  if (src == wire) return dtype_info(src).kind != VK_NONE && dtype_info(src).kind != VK_STRING;
  return (wire == DT_FLOAT && (src == DT_HALF || src == DT_BFLOAT16)) ? 1 : 0;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------
// wire-size arithmetic and header bytes
// ------------------------------------------------------------------------------------------------
static bool request_needs_deferred(const b200tfs_request& r);                  // varint_host.inc
static int deferred_arena_size(int32_t n, const b200tfs_request* reqs, const b200tfs_request_spec* specs, uint64_t* bytes);   // varint_host.inc

namespace {

constexpr uint64_t kProtoLimit = 0x7FFFFFFFull;  // protobuf's 2 GiB message limit

// model_spec's layout (framing.h writes it); `s` (may be null) adds signature_name and version_label
template <class Req>
int spec_layout(const Req& r, SpecLayout* S, const b200tfs_request_spec* s = nullptr) {
  if (r.model_name_len < 0 || (r.model_name_len && !r.model_name)) return fail(B200TFS_E_ARG, "bad model_name");
  *S = SpecLayout{};
  if (r.model_name_len) S->body += 1 + varint_len((uint64_t)r.model_name_len) + (uint64_t)r.model_name_len;
  if (r.has_version) {
    S->version_len = r.version ? 1 + varint_len((uint64_t)r.version) : 0;
    S->body += 2 + S->version_len;
  }
  if (!s) return B200TFS_OK;
  if (s->signature_len < 0 || (s->signature_len && !s->signature_name)) return fail(B200TFS_E_ARG, "bad signature_name");
  if (s->version_label_len > 0 && !s->version_label) return fail(B200TFS_E_ARG, "bad version_label");
  if (s->version_label_len >= 0 && r.has_version)
    return fail(B200TFS_E_ARG, "version and version_label are members of one oneof: set at most one of them");
  if ((uint64_t)s->signature_len > kProtoLimit || (s->version_label_len > 0 && (uint64_t)s->version_label_len > kProtoLimit))
    return fail(B200TFS_E_TOOBIG, "signature_name or version_label exceeds protobuf's 2 GiB limit");
  S->sig = s->signature_name; S->sig_len = (uint64_t)s->signature_len;
  S->label = s->version_label; S->label_len = s->version_label_len < 0 ? -1 : s->version_label_len;
  if (S->sig_len) S->body += 1 + varint_len(S->sig_len) + S->sig_len;
  if (S->label_len >= 0) S->body += 1 + varint_len((uint64_t)S->label_len) + (uint64_t)S->label_len;
  return B200TFS_OK;
}

// bytes of the output_filter run framing.h's write_output_filter writes for `s` (may be null)
int filter_len(const b200tfs_request_spec* s, uint64_t* len) {
  *len = 0;
  if (!s) return B200TFS_OK;
  if (s->n_output_filter < 0 || (s->n_output_filter && (!s->output_filter || !s->output_filter_len)))
    return fail(B200TFS_E_ARG, "bad output_filter");
  for (int64_t i = 0; i < s->n_output_filter; ++i) {
    const int64_t l = s->output_filter_len[i];
    if (l < 0 || (l && !s->output_filter[i])) return fail(B200TFS_E_ARG, "bad output_filter name %lld", (long long)i);
    *len += 1 + varint_len((uint64_t)l) + (uint64_t)l;
    if (*len > kProtoLimit) return fail(B200TFS_E_TOOBIG, "output_filter exceeds protobuf's 2 GiB limit");
  }
  return B200TFS_OK;
}

// `deferred`: lay out for b200tfs_encode_requests_async, which counts every packed-varint payload on the device whatever
// packed_len says; anywhere else such a payload must have been measured
int tensor_layout(const b200tfs_tensor& t, TensorLayout* L, std::vector<uint8_t>* hdr, bool deferred = false) {
  *L = TensorLayout{};   // layouts are reused from request to request (request_layout): no field may survive
  if (t.flags & B200TFS_F_PRESERIALIZED) {  // an already serialised TensorProto: all payload, no header
    if (t.packed_len > kProtoLimit) return fail(B200TFS_E_TOOBIG, "serialised TensorProto exceeds 2 GiB");
    L->n_elems = t.packed_len; L->payload_len = t.packed_len; L->header_len = 0; L->op = OP_COPY; L->varint = false;
    return B200TFS_OK;
  }
  if (t.rank < 0 || t.rank > 254) return fail(B200TFS_E_SHAPE, "rank %d outside [0, 254]", t.rank);
  if (t.rank && !t.dims) return fail(B200TFS_E_ARG, "dims is NULL");
  L->src_info = dtype_info(t.src_dtype);
  L->wire_info = dtype_info(t.wire_dtype);
  if (L->src_info.kind == VK_NONE || L->wire_info.kind == VK_NONE)
    return fail(B200TFS_E_DTYPE, "dtype %d -> %d is not in the TensorProto table", t.src_dtype, t.wire_dtype);
  if (L->src_info.kind == VK_STRING || L->wire_info.kind == VK_STRING)
    return fail(B200TFS_E_DTYPE, "DT_STRING tensors are assembled on the host (string_val is not a device payload)");
  if (!b200tfs_cast_supported(t.src_dtype, t.wire_dtype))
    return fail(B200TFS_E_DTYPE, "cast DT %d -> DT %d is not supported", t.src_dtype, t.wire_dtype);
  uint64_t n = 1;
  for (int i = 0; i < t.rank; ++i) {
    int64_t d = t.dims[i];
    if (d < 0) return fail(B200TFS_E_SHAPE, "negative dim %lld", (long long)d);
    if (d && n > kProtoLimit * 16 / (uint64_t)d) return fail(B200TFS_E_TOOBIG, "tensor too large for one protobuf message");
    n *= (uint64_t)d;
  }
  L->n_elems = n;
  const bool content = (t.flags & B200TFS_F_TENSOR_CONTENT) != 0;
  const bool cast = t.src_dtype != t.wire_dtype;
  uint32_t field;
  if (content) {
    field = F_CONTENT;
    L->payload_len = n * L->wire_info.elem_size;
    L->op = cast ? (t.src_dtype == DT_HALF ? OP_H2F : OP_B2F) : OP_COPY;
  } else {
    field = L->wire_info.field;
    switch (L->wire_info.kind) {
      case VK_FIXED:
        L->payload_len = n * L->wire_info.elem_size;
        if (cast) L->op = (t.src_dtype == DT_HALF) ? OP_H2F : OP_B2F;
        else L->op = (t.wire_dtype == DT_FLOAT && !(t.flags & B200TFS_F_KEEP_SNAN)) ? OP_QUIET_SRC : OP_COPY;
        break;
      case VK_BOOL:
        L->payload_len = n;
        L->op = OP_BOOL;
        break;
      default:  // VK_VARINT
        L->varint = true;
        if (n && !deferred && t.packed_len == 0)
          return fail(B200TFS_E_ARG, "varint dtype %d: packed_len not set, call b200tfs_measure first", t.wire_dtype);
        L->payload_len = n && !deferred ? t.packed_len : 0;
        break;
    }
  }
  if (L->payload_len > kProtoLimit) return fail(B200TFS_E_TOOBIG, "payload of %llu bytes exceeds protobuf's 2 GiB limit", (unsigned long long)L->payload_len);
  const uint64_t shape_len = shape_body_len(t.rank, t.dims);
  uint64_t hl = 1 + varint_len((uint64_t)(uint32_t)t.wire_dtype) + 1 + varint_len(shape_len) + shape_len;
  if (L->payload_len) hl += varint_len(tag_of(field, WT_LEN)) + varint_len(L->payload_len);
  L->header_len = hl; L->field = field; L->shape_len = shape_len;
  if (hdr) {   // one resize, then raw writes
    const size_t base = hdr->size();
    hdr->resize(base + hl);
    RawOut o{hdr->data() + base};
    write_tensor_header(o, t, *L);
    if ((uint64_t)(o.w - (hdr->data() + base)) != hl) return fail(B200TFS_E_ARG, "internal: header length mismatch");
  }
  return B200TFS_OK;
}

// key order (SURVEY 8a Q1).  UPB: bytewise on the common prefix; on a tie the LONGER key first.
int order_keys(int32_t n, const char* const* keys, const int64_t* lens, int32_t order, int32_t* perm) {
  for (int i = 0; i < n; ++i) perm[i] = i;
  if (order == B200TFS_ORDER_GIVEN) return B200TFS_OK;
  if (order != B200TFS_ORDER_UPB && order != B200TFS_ORDER_BYTES) return fail(B200TFS_E_ARG, "unknown key order %d", order);
  std::stable_sort(perm, perm + n, [&](int a, int b) {
    size_t la = (size_t)lens[a], lb = (size_t)lens[b];
    int c = memcmp(keys[a], keys[b], std::min(la, lb));
    if (c) return c < 0;
    if (la == lb) return false;
    return order == B200TFS_ORDER_UPB ? la > lb : la < lb;
  });
  return B200TFS_OK;
}

struct VarJob {  // one varint-packed payload (handled by the varint kernels after move_kernel)
  const uint8_t* src;
  uint8_t* dst;
  uint64_t n_elems;
  uint64_t packed_len;
  int32_t src_dtype;
};

// Accumulates the pieces of a batch of records into a plan image.
struct PlanBuilder {
  std::vector<MoveItem> items;
  std::vector<SmallItem> smalls;
  std::vector<uint8_t> blob;
  std::vector<VarJob> varjobs;
  uint64_t large_bytes = 0;
  const uint32_t* guard = nullptr;   // move_guarded_kernel: item i is stored only if guard[i / guard_div] != 0
  uint32_t guard_div = 1;
  bool independent = false;          // PlanHeader::independent

  void header(uint8_t* dst, size_t blob_off, size_t n) {
    // split long headers so one warp never walks more than kSmallMax bytes
    while (n) {
      uint32_t k = (uint32_t)std::min<size_t>(n, kSmallMax);
      smalls.push_back(SmallItem{(uint64_t)blob_off, dst, k, OP_COPY | OP_FLAG_BLOB, 0, 0});
      dst += k; blob_off += k; n -= k;
    }
  }
  // glen / gstride != 0: the source is a row of pieces (b200tfs_run with count > 1), gathered byte-exact
  void payload(const uint8_t* src, uint8_t* dst, uint64_t n_out, uint32_t op, uint32_t glen = 0, uint32_t gstride = 0) {
    if (!n_out) return;
    if (n_out <= kSmallMax) smalls.push_back(SmallItem{(uint64_t)(uintptr_t)src, dst, (uint32_t)n_out, op, glen, gstride});
    else { items.push_back(MoveItem{src, dst, n_out, op, 0, glen, gstride}); large_bytes += n_out; }
  }
};

// Tile size of a launch: about 8 tiles per SM, rounded up to whole 32 KB and capped at `max_tile`.
uint32_t pick_vec_per_tile(const b200tfs_ctx* c, uint64_t large_bytes, uint64_t max_tile) {
  uint64_t tile = c->tile_bytes_override;
  if (!tile) {
    uint64_t target_tiles = (uint64_t)c->sm_count * 8;
    tile = (large_bytes + target_tiles - 1) / target_tiles;
    tile = (tile + 32767) & ~32767ull;
    tile = std::min<uint64_t>(std::max<uint64_t>(tile, 32768), max_tile);
  }
  tile = std::max<uint64_t>(tile & ~31ull, 32);
  return (uint32_t)(tile / 16);
}

// Serialise the plan image (blob offsets inside SmallItems are rebased onto the image).  Small images travel in the kernel
// parameters unless `force_dev`: then - and for large images - the image is uploaded and *plan_dev points at it.
struct BuiltPlan {
  PlanHeader ph{};
  uint8_t inline_buf[kInlinePlanBytes];
  const uint8_t* host_img = nullptr;
  uint8_t* plan_dev = nullptr;   // nullptr: inline
  uint64_t image = 0;
  Slot* slot = nullptr;
};

int build_plan(b200tfs_ctx* c, PlanBuilder& pb, bool force_dev, BuiltPlan* bp) {
  // 32 KB per CTA: the vector paths keep all of it in flight at once (8 x 16 B per thread).  Measured on an H100 (C2 batch of
  // 256 x 4 MiB in one launch): 730 us at 32 KB tiles against 751 us at 64 KB and 766 us at 128 KB
  const uint32_t vpt = pick_vec_per_tile(c, pb.large_bytes, 32768);
  // tiles
  uint64_t n_tiles = 0;
  uint32_t uniform = 0;
  bool is_uniform = !pb.items.empty();
  for (auto& it : pb.items) {
    uint64_t t = tiles_for_host(it.n_out, vpt);
    if (n_tiles + t > 0x7FFFFFFFull) return fail(B200TFS_E_TOOBIG, "batch needs more than 2^31 tiles");
    it.n_tiles = (uint32_t)t;
    if (&it == &pb.items[0]) uniform = (uint32_t)t; else if (t != uniform) is_uniform = false;
    n_tiles += t;
  }
  if (!is_uniform) uniform = 0;
  PlanHeader& ph = bp->ph;
  ph = PlanHeader{};
  ph.n_items = (uint32_t)pb.items.size();
  ph.n_tiles = (uint32_t)n_tiles;
  ph.n_small = (uint32_t)pb.smalls.size();
  ph.uniform_tpi = uniform;
  ph.vec_per_tile = vpt;
  ph.guard = pb.guard; ph.guard_div = pb.guard_div ? pb.guard_div : 1u;
  ph.independent = pb.independent ? 1u : 0u;
  const PlanGeometry g = plan_geometry(pb.items.size(), uniform ? 0 : n_tiles, pb.smalls.size());
  ph.off_items = (uint32_t)g.off_items; ph.off_tiles = (uint32_t)g.off_tiles; ph.off_small = (uint32_t)g.off_small;
  Layout P{g.end};
  const uint64_t off_blob = P.take(pb.blob.size(), 1);
  const uint64_t image = P.take(0);
  if (image > 0xFFFFFFFFull) return fail(B200TFS_E_TOOBIG, "plan image larger than 4 GiB");
  bp->image = image;
  uint8_t* img;
  const bool inl = !force_dev && image <= kInlinePlanBytes;
  if (inl) img = bp->inline_buf;
  else {
    int rc = claim_slot(c, image, &bp->slot);
    if (rc) return rc;
    img = (uint8_t*)bp->slot->host.p;
  }
  bp->host_img = img;
  memcpy(img, &ph, sizeof ph);
  if (!pb.items.empty()) memcpy(img + ph.off_items, pb.items.data(), pb.items.size() * sizeof(MoveItem));
  if (!uniform && n_tiles) {
    TileRef* tr = (TileRef*)(img + ph.off_tiles);
    uint32_t g = 0;
    for (uint32_t i = 0; i < pb.items.size(); ++i)
      for (uint32_t t = 0; t < pb.items[i].n_tiles; ++t) tr[g++] = TileRef{i, t};
  }
  SmallItem* sm = (SmallItem*)(img + ph.off_small);
  for (size_t i = 0; i < pb.smalls.size(); ++i) {
    sm[i] = pb.smalls[i];
    if (sm[i].op & OP_FLAG_BLOB) sm[i].src += off_blob;
  }
  if (!pb.blob.empty()) memcpy(img + off_blob, pb.blob.data(), pb.blob.size());
  if (!inl) {
    int rc = upload_slot(c, bp->slot, image);
    if (rc) return rc;
    bp->plan_dev = (uint8_t*)bp->slot->dev.p;
  }
  return B200TFS_OK;
}

int launch_built_plan(b200tfs_ctx* c, BuiltPlan& bp) {
  CU(launch_move(bp.plan_dev, bp.host_img, (uint32_t)bp.image, bp.ph.n_tiles, bp.ph.n_small, c->stream));
  c->launches += 1;
  if (bp.slot && bp.slot->done && !c->capturing) { CU(cudaEventRecord(bp.slot->done, c->stream)); bp.slot->pending = true; }   // the kernel still reads the image
  return B200TFS_OK;
}

int launch_plan(b200tfs_ctx* c, PlanBuilder& pb) {
  if (pb.items.empty() && pb.smalls.empty()) return B200TFS_OK;
  BuiltPlan bp;
  int rc = build_plan(c, pb, false, &bp);
  if (rc) return rc;
  return launch_built_plan(c, bp);
}

// record placement: slots start 256-byte aligned, then padded so the record's largest payload
// starts 128-byte aligned (the vector path then needs no realignment for it)
inline uint64_t place_record(uint64_t cursor, uint64_t largest_payload_off) {
  uint64_t slot = (cursor + 255) & ~255ull;
  uint64_t pad = (128 - (largest_payload_off & 127)) & 127;
  return slot + pad;
}

// Lay one TensorProto at arena+rec_off; appends its pieces to the plan.  `hdr_prefix` bytes (entry
// framing) have already been appended to pb.blob starting at blob_mark and precede the proto header.
int plan_tensor(const b200tfs_tensor& t, const TensorLayout& L, uint8_t* dst_payload, PlanBuilder& pb) {
  if (!L.payload_len) return B200TFS_OK;
  if (L.varint) {
    pb.varjobs.push_back(VarJob{(const uint8_t*)t.data, dst_payload, L.n_elems, L.payload_len, t.src_dtype});
    return B200TFS_OK;
  }
  pb.payload((const uint8_t*)t.data, dst_payload, L.payload_len, L.op);
  return B200TFS_OK;
}

int run_varjobs(b200tfs_ctx* c, PlanBuilder& pb);  // varint.cpp part below

struct RequestLayout {
  std::vector<TensorLayout> tl;
  std::vector<int32_t> perm;
  std::vector<uint64_t> tp_len, entry_len;
  SpecLayout spec;
  const b200tfs_request_spec* s = nullptr;   // signature, label and output_filter (may be null)
  uint64_t tail = 0;          // bytes of the output_filter run behind the last input
  uint64_t total = 0;
  uint64_t prefix = 0;        // bytes in front of the message: gRPC's 5-byte frame header when asked for
  uint64_t largest_off = 0;
  std::vector<uint64_t> payload_off;
};

// Validates request r, orders its keys and lays it out.  `deferred` (b200tfs_encode_requests_async): packed-varint inputs are
// unmeasured, and the record's total - which then depends on lengths the device counts - is checked on the device.
int request_layout(const b200tfs_request& r, const b200tfs_request_spec* s, RequestLayout* R, bool deferred = false) {
  if (r.n_inputs < 0) return fail(B200TFS_E_ARG, "n_inputs < 0");
  if (r.n_inputs && !r.inputs) return fail(B200TFS_E_ARG, "inputs is NULL");
  int rc = spec_layout(r, &R->spec, s);
  if (rc) return rc;
  if ((rc = filter_len(s, &R->tail))) return rc;
  R->s = s;
  const int n = r.n_inputs;
  R->tl.resize(n); R->perm.resize(n); R->tp_len.resize(n); R->entry_len.resize(n); R->payload_off.resize(n);
  // (no heap traffic for the usual handful of inputs: this runs once per request of a batch)
  constexpr int kInline = 16;
  const char* keys_in[kInline];
  int64_t lens_in[kInline];
  std::vector<const char*> keys_v;
  std::vector<int64_t> lens_v;
  const char** keys = keys_in;
  int64_t* lens = lens_in;
  if (n > kInline) { keys_v.resize(n); lens_v.resize(n); keys = keys_v.data(); lens = lens_v.data(); }
  for (int i = 0; i < n; ++i) {
    if (r.inputs[i].key_len < 0 || (r.inputs[i].key_len && !r.inputs[i].key)) return fail(B200TFS_E_ARG, "bad key on input %d", i);
    keys[i] = r.inputs[i].key ? r.inputs[i].key : "";
    lens[i] = r.inputs[i].key_len;
  }
  if (n == 1 && (r.order == B200TFS_ORDER_GIVEN || r.order == B200TFS_ORDER_UPB || r.order == B200TFS_ORDER_BYTES)) R->perm[0] = 0;
  else rc = order_keys(n, keys, lens, r.order, R->perm.data());
  if (rc) return rc;
  if (r.flags & ~B200TFS_RF_GRPC_FRAME) return fail(B200TFS_E_ARG, "unknown request flags 0x%x", (unsigned)r.flags);
  R->prefix = (r.flags & B200TFS_RF_GRPC_FRAME) ? 5 : 0;
  uint64_t total = R->prefix + R->spec.field();
  uint64_t largest = 0;
  R->largest_off = 0;
  for (int j = 0; j < n; ++j) {
    const b200tfs_tensor& t = r.inputs[R->perm[j]];
    TensorLayout& L = R->tl[j];
    if ((rc = tensor_layout(t, &L, nullptr, deferred))) return rc;
    uint64_t tp = L.header_len + L.payload_len;
    if (tp > kProtoLimit) return fail(B200TFS_E_TOOBIG, "TensorProto of %llu bytes exceeds 2 GiB", (unsigned long long)tp);
    R->tp_len[j] = tp;
    uint64_t el = 1 + varint_len((uint64_t)t.key_len) + (uint64_t)t.key_len + 1 + varint_len(tp) + tp;
    R->entry_len[j] = el;
    uint64_t entry_hdr = 1 + varint_len(el) + 1 + varint_len((uint64_t)t.key_len) + (uint64_t)t.key_len + 1 + varint_len(tp);
    uint64_t payload_off = total + entry_hdr + L.header_len;
    R->payload_off[j] = payload_off;
    if (L.payload_len > largest) { largest = L.payload_len; R->largest_off = payload_off; }
    total += 1 + varint_len(el) + el;
  }
  total += R->tail;
  if (!deferred && total - R->prefix > kProtoLimit)
    return fail(B200TFS_E_TOOBIG, "PredictRequest of %llu bytes exceeds protobuf's 2 GiB limit", (unsigned long long)(total - R->prefix));
  R->total = total;
  return B200TFS_OK;
}

// write_request's view of request r for the host planner: the framing goes to the blob, and every payload closes the header run
// in front of it into the plan
struct PlannedRequest {
  const b200tfs_request& r;
  const RequestLayout& R;
  PlanBuilder& pb;
  uint8_t* w0;            // the request's framing in the blob
  size_t base;            // ... at this blob offset
  size_t mark;            // blob offset where the pending header run starts
  uint8_t* cursor;        // where that run will land
  void spec(RawOut& o) { write_model_spec(o, r, R.spec); }
  void tail(RawOut& o) { write_output_filter(o, R.s); }     // the trailing header run plan_request closes after the last payload
  void input(uint32_t j, b200tfs_tensor& t, TensorLayout& L) const { t = r.inputs[R.perm[j]]; L = R.tl[j]; }
  void payload(RawOut& o, uint32_t, const b200tfs_tensor& t, const TensorLayout& L) {
    if (!L.payload_len) return;
    const size_t at = base + (size_t)(o.w - w0), run = at - mark;
    pb.header(cursor, mark, run);
    cursor += run;
    plan_tensor(t, L, cursor, pb);
    cursor += L.payload_len;
    mark = at;
  }
};

// append the wire bytes of request r to the plan, record at arena + rec_off.  Every framing byte of the request is
// written into the blob with one resize and raw stores (this runs once per request of a batch); the tensor layouts are
// the ones request_layout computed.
int plan_request(const b200tfs_request& r, const RequestLayout& R, uint8_t* rec, PlanBuilder& pb) {
  uint64_t frame = R.total;
  for (int j = 0; j < r.n_inputs; ++j) frame -= R.tl[j].payload_len;
  const size_t base = pb.blob.size();
  pb.blob.resize(base + frame);
  uint8_t* const w0 = pb.blob.data() + base;
  RawOut o{w0};
  PlannedRequest q{r, R, pb, w0, base, base, rec};
  write_request(o, q, (uint32_t)r.n_inputs, R.prefix != 0, R.total - R.prefix);
  const size_t end = base + (size_t)(o.w - w0), run = end - q.mark;
  if (run) { pb.header(q.cursor, q.mark, run); q.cursor += run; }
  if ((uint64_t)(o.w - w0) != frame || (uint64_t)(q.cursor - rec) != R.total) return fail(B200TFS_E_ARG, "internal: request length mismatch");
  return B200TFS_OK;
}

}  // namespace

extern "C" {

int b200tfs_tensor_proto_size(const b200tfs_tensor* t, uint64_t* header_len, uint64_t* total_len) {
  if (!t) return fail(B200TFS_E_ARG, "tensor is NULL");
  TensorLayout L;
  int rc = tensor_layout(*t, &L, nullptr);
  if (rc) return rc;
  if (L.header_len + L.payload_len > kProtoLimit) return fail(B200TFS_E_TOOBIG, "TensorProto exceeds 2 GiB");
  if (header_len) *header_len = L.header_len;
  if (total_len) *total_len = L.header_len + L.payload_len;
  return B200TFS_OK;
}

int b200tfs_request_size(const b200tfs_request* r, uint64_t* total_len) { return b200tfs_request_size_spec(r, nullptr, total_len); }

int b200tfs_request_size_spec(const b200tfs_request* r, const b200tfs_request_spec* spec, uint64_t* total_len) {
  if (!r) return fail(B200TFS_E_ARG, "request is NULL");
  RequestLayout R;
  int rc = request_layout(*r, spec, &R);
  if (rc) return rc;
  if (total_len) *total_len = R.total;
  return B200TFS_OK;
}

int b200tfs_tensor_proto_header(const b200tfs_tensor* t, void* buf, uint64_t cap, uint64_t* len) {
  if (!t || !len) return fail(B200TFS_E_ARG, "NULL argument");
  TensorLayout L;
  std::vector<uint8_t> h;
  int rc = tensor_layout(*t, &L, &h);
  if (rc) return rc;
  *len = h.size();
  if (h.size() > cap) return fail(B200TFS_E_SIZE, "header needs %zu bytes", h.size());
  if (!h.empty()) memcpy(buf, h.data(), h.size());
  return B200TFS_OK;
}

int b200tfs_request_frame(const b200tfs_request* r, void* buf, uint64_t cap, uint64_t* frame_len, uint64_t* payload_off,
                          uint64_t* payload_len, int32_t* perm) {
  return b200tfs_request_frame_spec(r, nullptr, buf, cap, frame_len, payload_off, payload_len, perm);
}

int b200tfs_request_frame_spec(const b200tfs_request* r, const b200tfs_request_spec* spec, void* buf, uint64_t cap, uint64_t* frame_len,
                               uint64_t* payload_off, uint64_t* payload_len, int32_t* perm) {
  if (!r || !frame_len) return fail(B200TFS_E_ARG, "NULL argument");
  RequestLayout R;
  int rc = request_layout(*r, spec, &R);
  if (rc) return rc;
  PlanBuilder pb;  // planned against a NULL arena: only the blob (frame bytes in wire order) is used
  if ((rc = plan_request(*r, R, nullptr, pb))) return rc;
  *frame_len = pb.blob.size();
  for (int j = 0; j < r->n_inputs; ++j) {
    if (payload_off) payload_off[j] = R.payload_off[j];
    if (payload_len) payload_len[j] = R.tl[j].payload_len;
    if (perm) perm[j] = R.perm[j];
  }
  if (pb.blob.size() > cap) return fail(B200TFS_E_SIZE, "frame needs %zu bytes", pb.blob.size());
  if (!pb.blob.empty()) memcpy(buf, pb.blob.data(), pb.blob.size());
  return B200TFS_OK;
}

int b200tfs_order_keys(int32_t n, const char* const* keys, const int64_t* key_lens, int32_t order, int32_t* perm) {
  if (n < 0 || (n && (!keys || !key_lens || !perm))) return fail(B200TFS_E_ARG, "bad arguments");
  return order_keys(n, keys, key_lens, order, perm);
}

int b200tfs_tensor_arena_size(int32_t n, const b200tfs_tensor* tensors, uint64_t* bytes) {
  if (n < 0 || (n && !tensors) || !bytes) return fail(B200TFS_E_ARG, "bad arguments");
  uint64_t cursor = 0;
  for (int i = 0; i < n; ++i) {
    TensorLayout L;
    int rc = tensor_layout(tensors[i], &L, nullptr);
    if (rc) return rc;
    cursor = place_record(cursor, L.header_len) + L.header_len + L.payload_len;
  }
  *bytes = (cursor + 255) & ~255ull;
  return B200TFS_OK;
}

int b200tfs_request_arena_size(int32_t n, const b200tfs_request* reqs, uint64_t* bytes) {
  return b200tfs_request_arena_size_spec(n, reqs, nullptr, bytes);
}

int b200tfs_request_arena_size_spec(int32_t n, const b200tfs_request* reqs, const b200tfs_request_spec* specs, uint64_t* bytes) {
  if (n < 0 || (n && !reqs) || !bytes) return fail(B200TFS_E_ARG, "bad arguments");
  // a batch with an unmeasured packed-varint input (packed_len == 0) is sized for b200tfs_encode_requests_async: every record
  // gets a slot for its worst case; measured batches are sized exactly, as b200tfs_encode_requests lays them out
  bool deferred = false;
  for (int i = 0; i < n && !deferred; ++i) deferred = request_needs_deferred(reqs[i]);
  if (deferred) return deferred_arena_size(n, reqs, specs, bytes);
  uint64_t cursor = 0;
  RequestLayout R;
  for (int i = 0; i < n; ++i) {
    int rc = request_layout(reqs[i], specs ? specs + i : nullptr, &R);
    if (rc) return rc;
    cursor = place_record(cursor, R.largest_off) + R.total;
  }
  *bytes = (cursor + 255) & ~255ull;
  return B200TFS_OK;
}

int b200tfs_encode_tensor_protos(b200tfs_ctx* c, int32_t n, const b200tfs_tensor* tensors, void* arena_dev, uint64_t arena_cap,
                                 uint64_t* rec_off, uint64_t* rec_len) {
  if (!c || n < 0 || (n && (!tensors || !arena_dev || !rec_off || !rec_len))) return fail(B200TFS_E_ARG, "bad arguments");
  if ((uintptr_t)arena_dev & 255) return fail(B200TFS_E_ARG, "arena must be 256-byte aligned");
  CU(cudaSetDevice(c->device));
  PlanBuilder pb;
  uint64_t cursor = 0;
  for (int i = 0; i < n; ++i) {
    TensorLayout L;
    size_t mark = pb.blob.size();
    int rc = tensor_layout(tensors[i], &L, &pb.blob);
    if (rc) return rc;
    uint64_t total = L.header_len + L.payload_len;
    if (total > kProtoLimit) return fail(B200TFS_E_TOOBIG, "TensorProto exceeds 2 GiB");
    if (L.payload_len && !tensors[i].data) return fail(B200TFS_E_ARG, "tensor %d: data pointer is NULL", i);
    uint64_t off = place_record(cursor, L.header_len);
    if (off + total > arena_cap) return fail(B200TFS_E_SIZE, "arena too small: need %llu bytes", (unsigned long long)(off + total));
    uint8_t* rec = (uint8_t*)arena_dev + off;
    pb.header(rec, mark, L.header_len);
    if ((rc = plan_tensor(tensors[i], L, rec + L.header_len, pb))) return rc;
    rec_off[i] = off; rec_len[i] = total;
    cursor = off + total;
  }
  int rc = launch_plan(c, pb);
  if (rc) return rc;
  return run_varjobs(c, pb);
}

// lay the batch out in the arena and collect its pieces (b200tfs_encode_requests launches them at once, the pipelined host path in slices)
static int plan_requests(int32_t n, const b200tfs_request* reqs, const b200tfs_request_spec* specs, void* arena_dev, uint64_t arena_cap,
                         uint64_t* rec_off, uint64_t* rec_len, PlanBuilder& pb) {
  if (n > 16) {   // a batch: one allocation per table instead of a doubling series
    size_t inputs = 0;
    for (int i = 0; i < n; ++i) inputs += (size_t)std::max(reqs[i].n_inputs, 0);
    pb.items.reserve(inputs); pb.smalls.reserve(inputs + (size_t)n); pb.blob.reserve(64 * inputs + 48 * (size_t)n);
  }
  RequestLayout R;
  uint64_t cursor = 0;
  for (int i = 0; i < n; ++i) {
    int rc = request_layout(reqs[i], specs ? specs + i : nullptr, &R);
    if (rc) return rc;
    for (int j = 0; j < reqs[i].n_inputs; ++j)
      if (R.tl[j].payload_len && !reqs[i].inputs[R.perm[j]].data) return fail(B200TFS_E_ARG, "request %d: tensor data pointer is NULL", i);
    uint64_t off = place_record(cursor, R.largest_off);
    if (off + R.total > arena_cap) return fail(B200TFS_E_SIZE, "arena too small: need %llu bytes", (unsigned long long)(off + R.total));
    if ((rc = plan_request(reqs[i], R, (uint8_t*)arena_dev + off, pb))) return rc;
    rec_off[i] = off; rec_len[i] = R.total;
    cursor = off + R.total;
  }
  return B200TFS_OK;
}

static int encode_requests_spec(b200tfs_ctx* c, int32_t n, const b200tfs_request* reqs, const b200tfs_request_spec* specs, void* arena_dev,
                                uint64_t arena_cap, uint64_t* rec_off, uint64_t* rec_len) {
  if (!c || n < 0 || (n && (!reqs || !arena_dev || !rec_off || !rec_len))) return fail(B200TFS_E_ARG, "bad arguments");
  if ((uintptr_t)arena_dev & 255) return fail(B200TFS_E_ARG, "arena must be 256-byte aligned");
  CU(cudaSetDevice(c->device));
  PlanBuilder pb;
  int rc = plan_requests(n, reqs, specs, arena_dev, arena_cap, rec_off, rec_len, pb);
  if (rc) return rc;
  if ((rc = launch_plan(c, pb))) return rc;
  return run_varjobs(c, pb);
}

int b200tfs_encode_requests(b200tfs_ctx* c, int32_t n, const b200tfs_request* reqs, void* arena_dev, uint64_t arena_cap,
                            uint64_t* rec_off, uint64_t* rec_len) {
  return encode_requests_spec(c, n, reqs, nullptr, arena_dev, arena_cap, rec_off, rec_len);
}

// ---- decode ------------------------------------------------------------------------------------
static int parse_common(b200tfs_ctx* c, const void* arena_dev, int32_t n, const uint64_t* rec_off, const uint64_t* rec_len,
                        int32_t max_outputs, bool bare, b200tfs_output* outs, int32_t* n_outs, b200tfs_model_spec* specs,
                        int32_t* rec_status) {
  if (!c || n < 0 || (n && (!arena_dev || !rec_off || !rec_len || !outs || !rec_status))) return fail(B200TFS_E_ARG, "bad arguments");
  if (!bare && (max_outputs <= 0 || !n_outs || !specs)) return fail(B200TFS_E_ARG, "bad arguments");
  if (n == 0) return B200TFS_OK;
  if (c->capturing) return fail(B200TFS_E_ARG, "the two-phase parse synchronises and cannot be captured: use b200tfs_decode_responses");
  CU(cudaSetDevice(c->device));
  if (bare) max_outputs = 1;
  const uint64_t stride = bare ? 1 : (uint64_t)max_outputs + 1;  // responses: one scratch slot per record
  Layout B;   // rec_off | rec_len (uploaded) | outs | n_outs | specs | status | uint32 spill_used[n] (brought back)
  const uint64_t b_off = B.take(8ull * n), b_len = B.take(8ull * n);
  const uint64_t b_outs = B.take(sizeof(b200tfs_output) * (uint64_t)n * stride), b_nouts = B.take(4ull * n);
  const uint64_t b_specs = B.take(sizeof(b200tfs_model_spec) * (uint64_t)n), b_status = B.take(4ull * n);
  const uint64_t b_spill = B.take(4ull * n), total = B.end;
  int rc;
  if ((rc = grow_dev(c, c->scratch_dev, total))) return rc;
  if ((rc = grow_host(c, c->scratch_host, total))) return rc;
  uint8_t* h = (uint8_t*)c->scratch_host.p;
  uint8_t* d = (uint8_t*)c->scratch_dev.p;
  memcpy(h + b_off, rec_off, 8ull * n);
  memcpy(h + b_len, rec_len, 8ull * n);
  CU(cudaMemcpyAsync(d, h, b_outs, cudaMemcpyHostToDevice, c->stream));
  static_assert(sizeof(SpillEntry) == kSpillEntryBytes, "SpillEntry layout");
  // The walk runs with a spill area of spill_per_rec entries per record; a record that wants more says how many
  // (B200TFS_E_SPILL + spill_used) and the walk runs once more with that much - the count is exact, so twice at most.
  uint32_t per = c->spill_per_rec;
  c->spill_host.clear(); c->spill_last_n = 0; c->spill_last_per = 0;
  for (int attempt = 0;; ++attempt) {
    if ((rc = grow_dev(c, c->spill_dev, (uint64_t)n * per * sizeof(SpillEntry) + 16))) return rc;
    if (bare)
      CU(launch_parse_tensors((const uint8_t*)arena_dev, (const uint64_t*)(d + b_off), (const uint64_t*)(d + b_len), n,
                              (b200tfs_output*)(d + b_outs), (int32_t*)(d + b_status), c->spill_dev.p, per, (uint32_t*)(d + b_spill), c->stream));
    else
      CU(launch_parse_responses((const uint8_t*)arena_dev, (const uint64_t*)(d + b_off), (const uint64_t*)(d + b_len), n, max_outputs,
                                (b200tfs_output*)(d + b_outs), (int32_t*)(d + b_nouts), (b200tfs_model_spec*)(d + b_specs),
                                (int32_t*)(d + b_status), c->spill_dev.p, per, (uint32_t*)(d + b_spill), c->stream));
    c->launches += 1;
    CU(cudaMemcpyAsync(h + b_outs, d + b_outs, total - b_outs, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    const int32_t* st = (const int32_t*)(h + b_status);
    const uint32_t* used = (const uint32_t*)(h + b_spill);
    uint32_t want = 0, any = 0;
    bool again = false;
    for (int i = 0; i < n; ++i) { any |= used[i]; if (st[i] == B200TFS_E_SPILL) { again = true; want = std::max(want, used[i]); } }
    if (again && attempt < 2) {
      if ((uint64_t)n * want * sizeof(SpillEntry) > (1ull << 32)) return fail(B200TFS_E_TOOBIG, "spill area of %u entries x %d records", want, n);
      per = want;
      continue;
    }
    if (any) {   // bring the area over: unpack and the b200tfs_output_* accessors read it on the host
      c->spill_host.resize((size_t)n * per);
      CU(cudaMemcpyAsync(c->spill_host.data(), c->spill_dev.p, (size_t)n * per * sizeof(SpillEntry), cudaMemcpyDeviceToHost, c->stream));
      CU(cudaStreamSynchronize(c->stream));
      c->spill_last_n = n; c->spill_last_per = per;
    }
    break;
  }
  memcpy(rec_status, h + b_status, 4ull * n);
  for (int i = 0; i < n; ++i) if (rec_status[i] == B200TFS_E_SPILL) rec_status[i] = B200TFS_E_NONCANONICAL;   // cannot happen: the second walk had room
  if (bare) {
    memcpy(outs, h + b_outs, sizeof(b200tfs_output) * (uint64_t)n);
  } else {
    memcpy(n_outs, h + b_nouts, 4ull * n);
    memcpy(specs, h + b_specs, sizeof(b200tfs_model_spec) * (uint64_t)n);
    for (int i = 0; i < n; ++i) {
      int k = rec_status[i] == B200TFS_OK ? n_outs[i] : 0;
      memcpy(outs + (size_t)i * max_outputs, h + b_outs + sizeof(b200tfs_output) * (uint64_t)i * stride, sizeof(b200tfs_output) * (size_t)k);
    }
  }
  return B200TFS_OK;
}

// every value run of an output, in wire order: the inline ones, then the spilled ones of its map entry and value field
static int collect_runs(const b200tfs_ctx* c, const b200tfs_output& o, std::vector<b200tfs_run>& runs) {
  runs.clear();
  const uint32_t inl = std::min<uint32_t>(o.n_inline, B200TFS_MAX_RUNS);
  for (uint32_t k = 0; k < inl; ++k) runs.push_back(o.runs[k]);
  if ((uint32_t)o.n_runs > inl) {
    if (!(o.flags & B200TFS_OF_SPILLED) || (int32_t)o.spill_rec >= c->spill_last_n || c->spill_host.empty())
      return fail(B200TFS_E_ARG, "output lists %d value runs, %u inline, but the context holds no spill area for it (another parse ran since?)",
                  o.n_runs, inl);
    const SpillEntry* e = c->spill_host.data() + (size_t)o.spill_rec * c->spill_last_per;
    for (uint32_t k = 0; k < c->spill_last_per && (int)runs.size() < o.n_runs; ++k)
      if (e[k].kind == SPILL_RUN && e[k].seq == o.spill_seq && (int32_t)e[k].run.field == o.value_field) runs.push_back(e[k].run);
    if ((int)runs.size() != o.n_runs) return fail(B200TFS_E_ARG, "spill area does not hold the %d runs this output lists", o.n_runs);
  }
  return B200TFS_OK;
}

int b200tfs_output_runs(b200tfs_ctx* c, const b200tfs_output* o, b200tfs_run* runs, int32_t cap) {
  if (!c || !o || (cap > 0 && !runs) || cap < 0) return fail(B200TFS_E_ARG, "bad arguments");
  std::vector<b200tfs_run> all;
  int rc = collect_runs(c, *o, all);
  if (rc) return rc;
  for (int32_t k = 0; k < cap && k < (int32_t)all.size(); ++k) runs[k] = all[k];
  return B200TFS_OK;
}

int b200tfs_output_dims(b200tfs_ctx* c, const b200tfs_output* o, int64_t* dims, int32_t cap) {
  if (!c || !o || (cap > 0 && !dims) || cap < 0) return fail(B200TFS_E_ARG, "bad arguments");
  int32_t k = 0;
  for (; k < cap && k < o->rank && k < B200TFS_MAX_RANK; ++k) dims[k] = o->dims[k];
  if (o->rank > B200TFS_MAX_RANK && cap > B200TFS_MAX_RANK) {
    if ((int32_t)o->spill_rec >= c->spill_last_n || c->spill_host.empty())
      return fail(B200TFS_E_ARG, "rank %d output, but the context holds no spill area for it (another parse ran since?)", o->rank);
    const SpillEntry* e = c->spill_host.data() + (size_t)o->spill_rec * c->spill_last_per;
    for (uint32_t i = 0; i < c->spill_last_per && k < cap && k < o->rank; ++i)
      if (e[i].kind == SPILL_DIM && e[i].seq == o->spill_seq) dims[k++] = (int64_t)e[i].run.off;
    if (k < std::min(cap, o->rank)) return fail(B200TFS_E_ARG, "spill area does not hold the %d dims this output lists", o->rank);
  }
  return B200TFS_OK;
}

int b200tfs_parse_responses(b200tfs_ctx* c, const void* arena_dev, int32_t n, const uint64_t* rec_off, const uint64_t* rec_len,
                            int32_t max_outputs, b200tfs_output* outs, int32_t* n_outs, b200tfs_model_spec* specs,
                            int32_t* rec_status) {
  return parse_common(c, arena_dev, n, rec_off, rec_len, max_outputs, false, outs, n_outs, specs, rec_status);
}

int b200tfs_parse_tensor_protos(b200tfs_ctx* c, const void* arena_dev, int32_t n, const uint64_t* rec_off, const uint64_t* rec_len,
                                b200tfs_output* outs, int32_t* rec_status) {
  return parse_common(c, arena_dev, n, rec_off, rec_len, 1, true, outs, nullptr, nullptr, rec_status);
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------
// unpack
// ------------------------------------------------------------------------------------------------
namespace {

struct VarDecodeJob {
  const uint8_t* src[B200TFS_MAX_RUNS];
  uint64_t len[B200TFS_MAX_RUNS];
  int n_chunks;
  uint8_t* dst;
  uint64_t n_elems;
  int32_t dtype;
  int32_t out_index;
  bool half_as_value;
  bool pad_edge;   // fewer values than elements: repeat the last one (B200TFS_OF_PAD_EDGE)
};

int run_vardecode(b200tfs_ctx* c, std::vector<VarDecodeJob>& jobs, int32_t* status);  // below

}  // namespace

// after a synchronise: the status words the varint decoder left in pinned memory -> the caller's array
static void collect_varint_status(b200tfs_ctx* c, int32_t* status) {
  if (status)
    for (size_t i = 0; i < c->pending_status.size(); ++i) status[c->pending_status[i]] = ((const int32_t*)c->scratch_host.p)[i];
  c->pending_status.clear();
}

// wait = false: everything is enqueued, nothing synchronised; the caller synchronises and calls collect_varint_status
static int unpack_outputs_impl(b200tfs_ctx* c, const void* arena_dev, int32_t m, const b200tfs_output* outs, const uint64_t* out_rec_off,
                               void* const* dst_dev, const int32_t* dst_dtype, int32_t* status, bool wait) {
  if (!c || m < 0 || (m && (!arena_dev || !outs || !dst_dev))) return fail(B200TFS_E_ARG, "bad arguments");
  CU(cudaSetDevice(c->device));
  PlanBuilder pb;
  std::vector<VarDecodeJob> vjobs;
  struct Fill { uint8_t* dst; uint32_t elem_size; uint64_t have, n_elems; };
  std::vector<Fill> fills;   // B200TFS_OF_PAD_EDGE on fixed-width outputs: pad once the values are in place
  // value runs of every output (inline + spilled).  Packed-varint outputs whose values lie in strided runs (rows of unpacked
  // elements) or in more runs than a decode job lists are first GATHERED into one contiguous stream - the concatenation of
  // the pieces is itself a packed varint stream - and decoded from there.
  std::vector<std::vector<b200tfs_run>> all_runs(m);
  uint64_t gather_bytes = 0;
  for (int j = 0; j < m; ++j) {
    const b200tfs_output& o = outs[j];
    if (!o.n_elems || o.n_runs == 0) continue;
    int rc = collect_runs(c, o, all_runs[j]);
    if (rc) return rc;
    const uint32_t kind = dtype_info(o.dtype).kind;
    if (kind == VK_VARINT || kind == VK_BOOL) {
      bool plain = all_runs[j].size() <= (size_t)B200TFS_MAX_RUNS;
      uint64_t bytes = 0;
      for (const b200tfs_run& r : all_runs[j]) { plain = plain && r.count == 1; bytes += (uint64_t)r.len * r.count; }
      if (!plain) gather_bytes = ((gather_bytes + 15) & ~15ull) + bytes;
    }
  }
  if (gather_bytes) { int rc = grow_dev(c, c->gather_dev, gather_bytes + 64); if (rc) return rc; }
  uint64_t gather_cur = 0;
  for (int j = 0; j < m; ++j) {
    const b200tfs_output& o = outs[j];
    const std::vector<b200tfs_run>& runs = all_runs[j];
    const uint8_t* w = (const uint8_t*)arena_dev + (out_rec_off ? out_rec_off[j] : 0);  // table offsets are record-relative
    if (status) status[j] = B200TFS_OK;
    if (!o.n_elems) continue;
    const bool content_only = o.n_runs == 0 && o.content_len && o.content_len == o.dst_bytes;
    // TF's MakeNdarray convention, asked for by the caller.  For packed varints the table cannot know the element count
    // (status OK unless there are fewer value BYTES than elements): the flag then tells the decode kernels to tolerate it.
    const bool pad = (o.flags & B200TFS_OF_PAD_EDGE) &&
                     (o.status == B200TFS_E_SHAPE || (o.status == B200TFS_OK && (o.flags & B200TFS_OF_VARINT)));
    if (o.status != B200TFS_OK && !content_only && !pad)
      return fail(B200TFS_E_ARG, "output %d was tabulated with status %d: nothing to unpack", j, o.status);
    DtypeInfo di = dtype_info(o.dtype);
    if (di.kind == VK_NONE || di.kind == VK_STRING) return fail(B200TFS_E_DTYPE, "output %d: dtype %d has no device payload", j, o.dtype);
    if (!dst_dev[j]) return fail(B200TFS_E_ARG, "output %d: dst is NULL", j);
    int32_t want = dst_dtype ? dst_dtype[j] : o.dtype;
    const bool half_as_value = (want == B200TFS_DT_HALF_REFQUIRK && o.dtype == DT_HALF);
    if (half_as_value) want = DT_HALF;
    uint8_t* dst = (uint8_t*)dst_dev[j];
    if (pad && want != o.dtype) return fail(B200TFS_E_DTYPE, "output %d: cast together with padding is not supported", j);
    if (o.n_runs == 0 && pad && !content_only) {   // no values at all: zeros
      CU(cudaMemsetAsync(dst, 0, o.dst_bytes, c->stream));
      continue;
    }
    if (o.n_runs == 0) {
      // tolerant path chosen by the caller: raw little-endian bytes from tensor_content
      if (o.content_len != o.dst_bytes) return fail(B200TFS_E_SHAPE, "output %d: no values (tensor_content %llu bytes, need %llu)", j,
                                                     (unsigned long long)o.content_len, (unsigned long long)o.dst_bytes);
      if (want != o.dtype) return fail(B200TFS_E_DTYPE, "output %d: cast from tensor_content is not supported", j);
      pb.payload(w + o.content_off, dst, o.content_len, OP_COPY);
      continue;
    }
    if (di.kind == VK_FIXED) {
      uint32_t op;
      uint32_t num = 1, den = 1;  // dst bytes per src byte
      if (want == o.dtype) op = (o.dtype == DT_FLOAT) ? OP_QUIET_DST : OP_COPY;
      else if (o.dtype == DT_FLOAT && want == DT_HALF) { op = OP_F2H; den = 2; }
      else if (o.dtype == DT_FLOAT && want == DT_BFLOAT16) { op = OP_F2B; den = 2; }
      else return fail(B200TFS_E_DTYPE, "output %d: cast DT %d -> DT %d is not supported", j, o.dtype, want);
      uint64_t run = 0;
      for (const b200tfs_run& r : runs) {
        const uint64_t bytes = (uint64_t)r.len * r.count * num / den;
        if (r.count == 1) pb.payload(w + r.off, dst + run, bytes, op);
        else pb.payload(w + r.off, dst + run, bytes, op, r.len, r.stride);
        run += bytes;
      }
      if (pad) {
        if (run % di.elem_size || run > o.dst_bytes) return fail(B200TFS_E_SHAPE, "output %d: %llu value bytes for a tensor of %llu", j,
                                                                  (unsigned long long)run, (unsigned long long)o.dst_bytes);
        fills.push_back(Fill{dst, di.elem_size, run / di.elem_size, o.n_elems});
      }
    } else {  // packed varints (incl. bool_val)
      if (want != o.dtype) return fail(B200TFS_E_DTYPE, "output %d: cast on varint dtypes is not supported", j);
      VarDecodeJob vj{};
      bool plain = runs.size() <= (size_t)B200TFS_MAX_RUNS;
      for (const b200tfs_run& r : runs) plain = plain && r.count == 1;
      if (plain) {
        vj.n_chunks = (int)runs.size();
        for (size_t k = 0; k < runs.size(); ++k) { vj.src[k] = w + runs[k].off; vj.len[k] = runs[k].len; }
      } else {   // gather the pieces into one stream (same launch as the fixed-width moves, ahead of the decode kernels)
        gather_cur = (gather_cur + 15) & ~15ull;
        uint8_t* g = (uint8_t*)c->gather_dev.p + gather_cur;
        uint64_t at = 0;
        for (const b200tfs_run& r : runs) {
          const uint64_t bytes = (uint64_t)r.len * r.count;
          if (r.count == 1) pb.payload(w + r.off, g + at, bytes, OP_COPY);
          else pb.payload(w + r.off, g + at, bytes, OP_COPY, r.len, r.stride);
          at += bytes;
        }
        gather_cur += at;
        vj.n_chunks = 1; vj.src[0] = g; vj.len[0] = at;
      }
      vj.dst = dst; vj.n_elems = o.n_elems; vj.dtype = o.dtype; vj.out_index = j; vj.half_as_value = half_as_value; vj.pad_edge = pad;
      vjobs.push_back(vj);
    }
  }
  int rc = launch_plan(c, pb);
  if (rc) return rc;
  for (const Fill& f : fills) { CU(launch_fill_edge(f.dst, f.elem_size, f.have, nullptr, f.n_elems, c->stream)); c->launches += 1; }
  c->pending_status.clear();
  if (!vjobs.empty()) {
    if ((rc = run_vardecode(c, vjobs, status))) return rc;
  }
  if (status && wait) {
    CU(cudaStreamSynchronize(c->stream));
    collect_varint_status(c, status);
  }
  return B200TFS_OK;
}

extern "C" int b200tfs_unpack_outputs(b200tfs_ctx* c, const void* arena_dev, int32_t m, const b200tfs_output* outs,
                                      const uint64_t* out_rec_off, void* const* dst_dev, const int32_t* dst_dtype, int32_t* status) {
  return unpack_outputs_impl(c, arena_dev, m, outs, out_rec_off, dst_dev, dst_dtype, status, true);
}

// ------------------------------------------------------------------------------------------------
// fused single-launch decode + CUDA graph capture
// ------------------------------------------------------------------------------------------------
namespace {
struct FusedLayout { uint64_t outs, nouts, specs, status, vstatus, total; };
FusedLayout fused_layout(int32_t n) {
  Layout R;
  FusedLayout L;
  L.outs = R.take(sizeof(b200tfs_output) * (uint64_t)n * kFusedMaxOutputs);
  L.nouts = R.take(4ull * n);
  L.specs = R.take(sizeof(b200tfs_model_spec) * (uint64_t)n);
  L.status = R.take(4ull * n);
  L.vstatus = R.take(4ull * n * kFusedMaxOutputs);     // b200tfs_set_decode_varints: one status word per (record, output) slot
  L.total = R.end;
  return L;
}

// Layout of the device tables of the varint outputs of a single-launch decode (VarPlan), for n records and tile_cap tiles
struct VarPlanLayout { uint64_t jobs, segs, tile_seg, tile_val, group_sum, total, status, n_tiles, bytes; };
VarPlanLayout var_plan_layout(uint64_t n, uint64_t tile_cap) {
  const uint64_t slots = n * kFusedMaxOutputs;
  Layout R;
  VarPlanLayout V;
  V.jobs = R.take(slots * sizeof(VarJobDev));
  V.segs = R.take(slots * B200TFS_MAX_RUNS * sizeof(VarSeg));
  V.tile_seg = R.take(4 * tile_cap);
  V.tile_val = R.take(4 * tile_cap);
  V.group_sum = R.take(4 * (tile_cap / kVarGroupTiles + slots + 2));
  V.total = R.take(8 * slots);
  V.status = R.take(4 * slots);
  V.n_tiles = R.take(16);
  V.bytes = R.end;
  return V;
}

// b200tfs_encode_requests_async / b200tfs_encode_example_requests_async leave rec_off[n] | rec_len[n] | status[n] in pinned
// memory (enc_host), where b200tfs_encode_results reads them
struct EncResultsLayout { uint64_t rec_off, rec_len, status, bytes; };
EncResultsLayout enc_results_layout(uint64_t n) {
  Layout R;
  EncResultsLayout E;
  E.rec_off = R.take(8 * n);
  E.rec_len = R.take(8 * n);
  E.status = R.take(4 * n);
  E.bytes = R.end;
  return E;
}

// Point the pointers a launch writes its results through at enc_host, grown for n requests
int bind_enc_results(b200tfs_ctx* c, int32_t n, uint64_t** rec_off, uint64_t** rec_len, int32_t** status) {
  const EncResultsLayout E = enc_results_layout((uint64_t)n);
  int rc = grow_host(c, c->enc_host, E.bytes);
  if (rc) return rc;
  uint8_t* rh = (uint8_t*)c->enc_host.p;
  *rec_off = (uint64_t*)(rh + E.rec_off); *rec_len = (uint64_t*)(rh + E.rec_len); *status = (int32_t*)(rh + E.status);
  return B200TFS_OK;
}
}  // namespace

extern "C" {

// take over the template a kernel left in pinned memory, if it is newer than what the host knows (stream must be idle)
static void adopt_pinned_template(b200tfs_ctx* c) {
  if (!c->tpl_pinned) return;
  const TplInline& p = *c->tpl_pinned;
  // newer than what the host knows - valid or not: a record 0 that could not be learnt retires the old template too
  if (p.head.serial && (int32_t)(p.head.serial - c->tpl_known.head.serial) > 0) c->tpl_known = p;
}

// tile size of a decode launch over `wire_total` bytes: every CTA of the fused kernel first verifies the record's framing, so
// big batches get fatter tiles than the plain move (up to 64 KB, two staged chunks), though not much fatter: on an H100 the C2
// batch decode (256 x 4 MiB in one launch) took 724 us at 64 KB tiles against 740 us at 128 KB and 751 us at 256 KB
static uint32_t decode_vpt(const b200tfs_ctx* c, int32_t n, const uint64_t* rec_len) {
  uint64_t wire_total = 0;
  for (int i = 0; i < n; ++i) wire_total += rec_len[i];
  return pick_vec_per_tile(c, c->decode_cast ? wire_total / 2 : wire_total, 65536);
}

// The parse walk (walker.h) of one record that lies in host memory, up to `max` outputs.  A record the walker's 32-bit cursor
// cannot hold is B200TFS_E_PARSE, as the kernels find it.  `cur` (optional) is left where the walk ended.
static int walk_host_record(const void* rec, uint64_t len, int max, b200tfs_output* outs, int* cnt, b200tfs_model_spec* spec,
                            SpillArea sp = SpillArea{nullptr, 0u, 0u}, Cursor* cur = nullptr) {
  if (len > 0x7FFFFFFFull) return B200TFS_E_PARSE;
  Cursor own;
  Cursor& k = cur ? *cur : own;
  cur_open_host(k, (const uint8_t*)rec, (uint32_t)len);
  return walk_response(k, max, outs, cnt, spec, sp);
}

// Walk record 0 on the host (its bytes are in host memory) and build its template: the launch that follows then takes the
// template path from its first CTA on.  Returns false when the record does not qualify (the kernel will walk it).
static bool host_template(const uint8_t* rec0, uint64_t len, uint32_t vpt, uint64_t dst_stride, uint32_t serial, uint32_t cast, uint32_t varints,
                          Template* T) {
  T->in.head.valid = 0;
  if (!rec0 || len == 0) return false;
  b200tfs_output outs[kFusedMaxOutputs + 1];
  b200tfs_model_spec spec;
  int cnt = 0;
  Cursor cur;
  const int st = walk_host_record(rec0, len, kFusedMaxOutputs, outs, &cnt, &spec, SpillArea{nullptr, 0u, 0u}, &cur);
  if (st != B200TFS_OK) return false;
  const uint64_t used = tpl_layout_outputs(outs, cnt, dst_stride, cast, varints);
  for (int k = 0; k < cnt; ++k) if (outs[k].status == B200TFS_E_SIZE) return false;
  // the kernel's own check: the chunks' tiles must fit the budget the launch gives the record
  tpl_learn(T, cur, (uint32_t)len, outs, cnt, spec, st, vpt, (used + 255) & ~255ull, serial, cast, varints);
  return T->in.head.valid != 0;
}

// Slot bytes the single-launch decode lays out for host-resident records (the same walk and layout rule, with no stride limit and
// no cast, which can only shrink a range): the most any record uses, and how many varint ranges the batch has
int b200tfs_decode_slot_bytes(const void* wire_host, int32_t n, const uint64_t* rec_off, const uint64_t* rec_len, int32_t varints,
                              uint64_t* slot_bytes, int32_t* n_varint_outputs) {
  if (n < 0 || (n && (!wire_host || !rec_off || !rec_len)) || !slot_bytes) return fail(B200TFS_E_ARG, "bad arguments");
  uint64_t most = 0;
  int32_t nv = 0;
  for (int i = 0; i < n; ++i) {
    b200tfs_output outs[kFusedMaxOutputs + 1];
    b200tfs_model_spec spec;
    int cnt = 0;
    // a record the launch rejects (malformed, or too long for the walker) gets no slot bytes
    if (walk_host_record((const uint8_t*)wire_host + rec_off[i], rec_len[i], kFusedMaxOutputs, outs, &cnt, &spec) != B200TFS_OK) continue;
    most = std::max(most, tpl_layout_outputs(outs, cnt, ~0ull, 0u, varints ? 1u : 0u));
    for (int k = 0; k < cnt && varints; ++k)
      if (outs[k].status == B200TFS_OK && outs[k].n_elems && dtype_info(outs[k].dtype).kind != VK_FIXED && tpl_gets_range(1u, outs[k].dtype))
        ++nv;
  }
  *slot_bytes = most;
  if (n_varint_outputs) *n_varint_outputs = nv;
  return B200TFS_OK;
}

// The packed-varint outputs of a table a decode launch published: vdec_plan_kernel builds their decode tables in the region `vd`
// (var_plan_layout(vp.n, vp.tile_cap)), then the count and emit kernels run over them.  `vp` comes with the table, the wire and
// the destinations set; rec_off is the host's copy of the record offsets.  vp.status receives the per-slot statuses.  `pad`: the
// padded decode's element placement (VarPadMap).
static int launch_varint_tail(b200tfs_ctx* c, VarPlan& vp, uint8_t* vd, const uint64_t* rec_off, const VarPadMap* pad = nullptr) {
  const VarPlanLayout V = var_plan_layout(vp.n, vp.tile_cap);
  if (vp.n <= (uint32_t)kFusedInlineRecs) for (uint32_t i = 0; i < vp.n; ++i) vp.off_inl[i] = rec_off[i];
  vp.jobs = (VarJobDev*)(vd + V.jobs); vp.segs = (VarSeg*)(vd + V.segs); vp.tile_seg = (uint32_t*)(vd + V.tile_seg);
  vp.tile_val = (uint32_t*)(vd + V.tile_val); vp.group_sum = (uint32_t*)(vd + V.group_sum);
  vp.total = (unsigned long long*)(vd + V.total); vp.status = (int32_t*)(vd + V.status); vp.n_tiles = (uint32_t*)(vd + V.n_tiles);
  CU(launch_vdec_plan(vp, c->stream));
  VarTables tb{};
  tb.segs = vp.segs; tb.tile_seg = vp.tile_seg; tb.jobs = vp.jobs; tb.n_tiles = vp.tile_cap; tb.n_tiles_dev = vp.n_tiles;
  CU(launch_vdec_dev(tb, (uint32_t)c->sm_count * 4, c->stream, pad));
  c->launches += 3;
  return B200TFS_OK;
}

// What the varint decode found for one output slot of the table (kVarSlotIdle: a slot it did not take, left as tabulated)
static void fold_varint_status(b200tfs_output& o, int32_t s) {
  if (s == kVarSlotIdle) return;
  o.status = s;
  o.flags |= B200TFS_OF_DEVICE_VARINT;
}

// the pipelined host decode of ONE record: launch k covers tiles [tile_lo[k], tile_lo[k+1]) of the full grid (the last one also the
// slack CTAs behind them), waits for before[k] and is followed by after[k] on the context's stream
struct DecodeSlices {
  int K = 0;
  uint32_t tile_lo[b200tfs_ctx::kPipeMax + 1] = {};
  cudaEvent_t* before = nullptr;
  cudaEvent_t* after = nullptr;
};

// host_tpl: the template of record 0 as the HOST walked it, when the caller has the record's bytes (the *_host entry points), else nullptr
static int decode_launch(b200tfs_ctx* c, const void* arena_dev, int32_t n, const uint64_t* rec_off, const uint64_t* rec_len, void* dst_dev,
                         uint64_t dst_stride, uint32_t vpt, const Template* host_tpl, const DecodeSlices* sl = nullptr) {
  const uint64_t tile_bytes = 16ull * vpt;
  FusedLayout L = fused_layout(n);
  int rc;
  if ((rc = grow_host(c, c->fused_host, L.total))) return rc;
  // varint outputs (b200tfs_set_decode_varints): tables sized from a bound the host knows, before anything is queued
  uint64_t var_tile_cap = 0;
  if (c->decode_varints) {
    for (int i = 0; i < n; ++i) var_tile_cap += var_record_tile_bound(rec_len[i]);
    if (var_tile_cap > 0x7FFFFFFFull) return fail(B200TFS_E_TOOBIG, "batch needs more than 2^31 varint tiles");
    if ((rc = grow_dev(c, c->vdec_dev, var_plan_layout((uint64_t)n, var_tile_cap).bytes))) return rc;
  }
  if (!c->tpl_dev) {
    if (c->capturing) return fail(B200TFS_E_ARG, "run b200tfs_decode_responses once before capturing it");
    CU(cudaMalloc(&c->tpl_dev, 2 * sizeof(Template) + 64));   // + the three path counters (b200tfs_decode_stats)
    CU(cudaMemsetAsync(c->tpl_dev, 0, 2 * sizeof(Template) + 64, c->stream));
    CU(cudaHostAlloc((void**)&c->tpl_pinned, sizeof(TplInline), cudaHostAllocPortable | cudaHostAllocMapped));
    memset(c->tpl_pinned, 0, sizeof(TplInline));
  }
  FusedParams fp{};
  fp.w = (const uint8_t*)arena_dev; fp.dst = (uint8_t*)dst_dev; fp.dst_stride = dst_stride; fp.n = n; fp.vpt = vpt;
  fp.tpl_read = (const Template*)c->tpl_dev + (c->tpl_flip & 1);
  fp.tpl_write = (Template*)c->tpl_dev + ((c->tpl_flip & 1) ^ 1);
  c->tpl_flip ^= 1;
  fp.tpl_pinned = c->tpl_pinned;
  fp.stats = (unsigned long long*)((uint8_t*)c->tpl_dev + 2 * sizeof(Template));
  if (++c->serial == 0) c->serial = 1;
  fp.serial = c->serial;
  fp.cast = c->decode_cast;
  fp.varints = c->decode_varints;
  fp.tpli.head.valid = 0;
  if (host_tpl && host_tpl->in.head.valid) {
    if (vpt <= kStageVecsHost) {   // the single-response / small-batch kernel takes its template from the parameters when the host has one
      // this launch's device template IS the host's walk of record 0: upload it where the kernel reads it
      Slot* slot;
      if ((rc = claim_slot(c, sizeof(Template), &slot))) return rc;
      memcpy(slot->host.p, host_tpl, sizeof(Template));
      CU(cudaMemcpyAsync((void*)fp.tpl_read, slot->host.p, sizeof(Template), cudaMemcpyHostToDevice, c->stream));
      if (slot->done) { CU(cudaEventRecord(slot->done, c->stream)); slot->pending = true; }
      c->tpl_known = host_tpl->in;
      if (!c->opt_no_inline) fp.tpli = host_tpl->in;
    }
  } else {
    // the pinned copy is current once the previous decode launch of this context has completed (the stream itself may
    // well be busy again: the caller's own copy of the next response usually precedes this call)
    if (!c->capturing && (!c->tpl_event_pending || cudaEventQuery(c->tpl_event) == cudaSuccess)) { c->tpl_event_pending = false; adopt_pinned_template(c); }
    const TplHead& h = c->tpl_known.head;
    if (vpt <= kStageVecsHost && !c->opt_no_inline && h.valid && h.rec_len == rec_len[0] && h.vpt == vpt && h.cast == fp.cast &&
        h.varints == fp.varints && h.dst_need <= dst_stride)
      fp.tpli = c->tpl_known;
  }
  // CTAs per record: a record of the length the host knows a template for gets that template's tiles + the publishing CTA + one
  // spare; any other record ceil(len / tile) + kFusedSlackTiles (its values may lie in several chunks, each rounding up).  With
  // the flat slack, 8 of the 9 CTAs of a 4 KB response and 137 of the 265 of a narrowed 16 MiB one had no tile.  Should a record
  // of that length carry OTHER framing that needs more tiles, its status says so (B200TFS_E_NONCANONICAL, b200tfs.h).
  const TplHead& kh = (host_tpl && host_tpl->in.head.valid) ? host_tpl->in.head : c->tpl_known.head;
  const bool budget_known = kh.valid && kh.vpt == vpt && kh.cast == fp.cast && kh.varints == fp.varints && kh.dst_need <= dst_stride;
  auto ctas_for = [&](uint64_t len) -> uint64_t {
    if (budget_known && len == kh.rec_len) return (uint64_t)kh.total_tiles + 2;
    return (len + tile_bytes - 1) / tile_bytes + kFusedSlackTiles;
  };
  // the table is written by the kernel straight into pinned host memory (unified addressing): ~1 KB
  // of posted PCIe writes per record instead of a device table plus a copy node behind every launch
  uint8_t* d = (uint8_t*)c->fused_host.p;
  fp.outs = (b200tfs_output*)(d + L.outs); fp.n_outs = (int32_t*)(d + L.nouts);
  fp.specs = (b200tfs_model_spec*)(d + L.specs); fp.status = (int32_t*)(d + L.status);
  // lay the CTAs of a launch out: record r owns `per(len)` consecutive CTAs; small batches in the parameters, else one uploaded table
  auto lay_out = [&](FusedParams& q, auto&& per, uint64_t* grid_out) -> int {
    uint64_t grid = 0;
    if (n <= kFusedInlineRecs) {
      for (int i = 0; i < n; ++i) {
        q.inl.off[i] = rec_off[i]; q.inl.len[i] = rec_len[i]; q.inl.tile_start[i] = (uint32_t)grid;
        grid += per(rec_len[i]);
      }
      q.inl.tile_start[n] = (uint32_t)grid;
    } else {
      std::vector<uint32_t> ts(n + 1);
      for (int i = 0; i < n; ++i) { ts[i] = (uint32_t)grid; grid += per(rec_len[i]); }
      ts[n] = (uint32_t)grid;
      if (grid > 0x7FFFFFFFull) return fail(B200TFS_E_TOOBIG, "batch needs more than 2^31 tiles");
      Layout T;   // cta_rec[grid] | tile_start[n+1] | rec_off[n] | rec_len[n]
      const uint64_t o_cr = T.take(4 * grid), o_ts = T.take(4ull * (n + 1)), o_off = T.take(8ull * n), o_len = T.take(8ull * n);
      uint8_t* sd;
      int rc2 = upload_image(c, T.end, {{o_ts, ts.data(), 4ull * (n + 1)}, {o_off, rec_off, 8ull * n}, {o_len, rec_len, 8ull * n}}, &sd, nullptr,
                             [&](uint8_t* h, uint8_t*) {
                               uint32_t* cr = (uint32_t*)(h + o_cr);
                               for (int i = 0; i < n; ++i) for (uint32_t t = ts[i]; t < ts[i + 1]; ++t) cr[t] = (uint32_t)i;
                             });
      if (rc2) return rc2;
      q.cta_rec = (const uint32_t*)(sd + o_cr); q.tile_start = (const uint32_t*)(sd + o_ts);
      q.rec_off = (const uint64_t*)(sd + o_off); q.rec_len = (const uint64_t*)(sd + o_len);
    }
    if (grid > 0x7FFFFFFFull) return fail(B200TFS_E_TOOBIG, "batch needs more than 2^31 tiles");
    *grid_out = grid;
    return B200TFS_OK;
  };
  // The narrowing decode of a batch whose template the host knows, as three launches: the narrowing tile move runs twice as
  // long inside the fused kernel as in the generic move engine (it shares the walker's register cap there), so (1) two CTAs per record verify the
  // framing against the host's template - handed over in the parameters, the very one the plan below is built from - leave the
  // verdict in guard[r] and publish the table, (2) move_guarded_kernel moves every record's chunks from a host-built plan
  // and stores only where guard[r] says so, (3) the whole decode runs for the records still unguarded (none, normally: its
  // CTAs leave after one load).
  const TplInline* kt = (host_tpl && host_tpl->in.head.valid) ? &host_tpl->in : &c->tpl_known;
  bool split = fp.cast && !sl && budget_known && kh.total_tiles > 0 && (uint64_t)n * kh.rec_len >= (4ull << 20) && !c->opt_no_inline;
  for (int i = 0; i < n && split; ++i) split = rec_len[i] == kh.rec_len;
  if (split) {
    if ((rc = grow_dev(c, c->guard_dev, 4ull * n))) return rc;
    FusedParams fa = fp;
    fa.mode = 1; fa.guard = (uint32_t*)c->guard_dev.p; fa.tpli = *kt;
    uint64_t ga = 0;
    if ((rc = lay_out(fa, [](uint64_t) -> uint64_t { return 2; }, &ga))) return rc;
    CU(launch_decode_fused(fa, (uint32_t)ga, c->stream));
    PlanBuilder pb;
    uint32_t per_rec = 0;
    for (uint32_t q = 0; q < kt->head.n_chunks; ++q) if (kt->chunk[q].n_tiles) ++per_rec;
    pb.items.reserve((size_t)n * per_rec);
    for (int i = 0; i < n; ++i)
      for (uint32_t q = 0; q < kt->head.n_chunks; ++q) {
        const TplChunk& ch = kt->chunk[q];
        if (!ch.n_tiles) continue;
        const bool narrow = ch.op == OP_F2H || ch.op == OP_F2B;
        const uint64_t n_out = narrow ? ch.len / 2 : ch.len;
        pb.items.push_back(MoveItem{(const uint8_t*)arena_dev + rec_off[i] + ch.wire_off, (uint8_t*)dst_dev + (uint64_t)i * dst_stride + ch.dst_off, n_out,
                                    ch.op, 0, 0, 0});
        pb.large_bytes += n_out;
      }
    pb.guard = (const uint32_t*)c->guard_dev.p; pb.guard_div = per_rec;
    BuiltPlan bp;
    if ((rc = build_plan(c, pb, true, &bp))) return rc;
    CU(launch_move_guarded(bp.plan_dev, bp.ph.n_tiles, c->stream));
    if (bp.slot && bp.slot->done && !c->capturing) { CU(cudaEventRecord(bp.slot->done, c->stream)); bp.slot->pending = true; }
    c->launches += 2;
    fp.mode = 2; fp.guard = (uint32_t*)c->guard_dev.p;
  }
  uint64_t grid = 0;
  if ((rc = lay_out(fp, ctas_for, &grid))) return rc;
  if (sl) {
    if (n != 1 || !fp.tpli.head.valid) return fail(B200TFS_E_ARG, "internal: sliced decode without a host template");
    fp.trusted = 1;
    for (int k = 0; k < sl->K; ++k) {
      CU(cudaStreamWaitEvent(c->stream, sl->before[k], 0));
      fp.tile_bias = sl->tile_lo[k];
      const uint32_t end = (k + 1 == sl->K) ? (uint32_t)grid : sl->tile_lo[k + 1];
      CU(launch_decode_fused(fp, end - sl->tile_lo[k], c->stream));
      CU(cudaEventRecord(sl->after[k], c->stream));
      c->launches += 1;
    }
  } else {
    CU(launch_decode_fused(fp, (uint32_t)grid, c->stream));
    c->launches += 1;
  }
  c->fused_varints = fp.varints != 0;
  if (fp.varints) {
    // plan -> count -> emit over the table the launch(es) above published, then the per-output statuses to pinned memory
    VarPlan vp{};
    vp.outs = fp.outs; vp.n_outs = fp.n_outs; vp.rec_status = fp.status;
    vp.w = fp.w; vp.rec_off = fp.rec_off;
    vp.dst = fp.dst; vp.dst_stride = dst_stride; vp.n = (uint32_t)n; vp.tile_cap = (uint32_t)var_tile_cap;
    if ((rc = launch_varint_tail(c, vp, (uint8_t*)c->vdec_dev.p, rec_off))) return rc;
    CU(cudaMemcpyAsync((uint8_t*)c->fused_host.p + L.vstatus, vp.status, 4ull * n * kFusedMaxOutputs, cudaMemcpyDeviceToHost, c->stream));
  }
  c->fused_n = n;
  if (!c->capturing) { CU(cudaEventRecord(c->tpl_event, c->stream)); c->tpl_event_pending = true; }
  return B200TFS_OK;
}

int b200tfs_decode_responses(b200tfs_ctx* c, const void* arena_dev, int32_t n, const uint64_t* rec_off, const uint64_t* rec_len,
                             void* dst_dev, uint64_t dst_stride) {
  if (!c || n < 0 || (n && (!arena_dev || !rec_off || !rec_len || !dst_dev))) return fail(B200TFS_E_ARG, "bad arguments");
  if (n == 0) return B200TFS_OK;
  if (dst_stride & 255) return fail(B200TFS_E_ARG, "dst_stride must be a multiple of 256");
  if (!c->capturing) CU(cudaSetDevice(c->device));
  return decode_launch(c, arena_dev, n, rec_off, rec_len, dst_dev, dst_stride, decode_vpt(c, n, rec_len), nullptr);
}

int b200tfs_set_decode_cast(b200tfs_ctx* c, int32_t float_as) {
  if (!c) return fail(B200TFS_E_ARG, "ctx is NULL");
  if (c->capturing) return fail(B200TFS_E_ARG, "cannot change the decode cast during graph capture");
  if (float_as != 0 && float_as != DT_FLOAT && float_as != DT_HALF && float_as != DT_BFLOAT16)
    return fail(B200TFS_E_DTYPE, "DT_FLOAT outputs can leave as DT_FLOAT, DT_HALF or DT_BFLOAT16, not as dtype %d", float_as);
  c->decode_cast = (float_as == DT_HALF || float_as == DT_BFLOAT16) ? (uint32_t)float_as : 0u;
  return B200TFS_OK;
}

int b200tfs_set_decode_varints(b200tfs_ctx* c, int32_t on) {
  if (!c) return fail(B200TFS_E_ARG, "ctx is NULL");
  if (c->capturing) return fail(B200TFS_E_ARG, "cannot switch the varint decode during graph capture");
  c->decode_varints = on ? 1u : 0u;
  return B200TFS_OK;
}

int b200tfs_decode_results(b200tfs_ctx* c, int32_t n, b200tfs_output* outs, int32_t* n_outs, b200tfs_model_spec* specs,
                           int32_t* rec_status) {
  if (!c || n < 0) return fail(B200TFS_E_ARG, "bad arguments");
  if (c->capturing) return fail(B200TFS_E_ARG, "cannot collect results during graph capture");
  if (n > c->fused_n) return fail(B200TFS_E_ARG, "only %d records were decoded", c->fused_n);
  FusedLayout L = fused_layout(c->fused_n);
  CU(cudaStreamSynchronize(c->stream));
  const uint8_t* h = (const uint8_t*)c->fused_host.p;
  if (outs) memcpy(outs, h + L.outs, sizeof(b200tfs_output) * (uint64_t)n * kFusedMaxOutputs);
  if (outs && c->fused_varints) {   // what the varint decode found, for exactly the outputs vdec_plan_kernel took
    const int32_t* rs = (const int32_t*)(h + L.status);
    const int32_t* no = (const int32_t*)(h + L.nouts);
    const int32_t* vs = (const int32_t*)(h + L.vstatus);
    for (int r = 0; r < n; ++r)
      for (int k = 0; k < no[r] && rs[r] == B200TFS_OK && k < kFusedMaxOutputs; ++k)
        fold_varint_status(outs[(size_t)r * kFusedMaxOutputs + k], vs[(size_t)r * kFusedMaxOutputs + k]);
  }
  if (n_outs) memcpy(n_outs, h + L.nouts, 4ull * n);
  if (specs) memcpy(specs, h + L.specs, sizeof(b200tfs_model_spec) * (uint64_t)n);
  if (rec_status) memcpy(rec_status, h + L.status, 4ull * n);
  return B200TFS_OK;
}

int b200tfs_decode_stats(b200tfs_ctx* c, uint64_t* param_template, uint64_t* device_template, uint64_t* walked) {
  if (!c) return fail(B200TFS_E_ARG, "ctx is NULL");
  if (c->capturing) return fail(B200TFS_E_ARG, "cannot read the counters during graph capture");
  unsigned long long v[3] = {0, 0, 0};
  if (c->tpl_dev) {
    CU(cudaSetDevice(c->device));
    CU(cudaMemcpyAsync(v, (uint8_t*)c->tpl_dev + 2 * sizeof(Template), sizeof v, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
  }
  if (param_template) *param_template = v[0];
  if (device_template) *device_template = v[1];
  if (walked) *walked = v[2];
  return B200TFS_OK;
}

int b200tfs_capture_begin(b200tfs_ctx* c) {
  if (!c) return fail(B200TFS_E_ARG, "ctx is NULL");
  if (c->capturing) return fail(B200TFS_E_ARG, "already capturing");
  CU(cudaSetDevice(c->device));
  CU(cudaStreamSynchronize(c->stream));
  adopt_pinned_template(c);   // captured single-response decodes carry the template known now in their parameters
  for (auto& s : c->slots) s.pending = false;
  CU(cudaStreamBeginCapture(c->stream, cudaStreamCaptureModeRelaxed));
  c->capturing = true;
  return B200TFS_OK;
}

int b200tfs_capture_end(b200tfs_ctx* c, void** graph_exec) {
  if (!c || !graph_exec) return fail(B200TFS_E_ARG, "NULL argument");
  if (!c->capturing) return fail(B200TFS_E_ARG, "not capturing");
  c->capturing = false;
  cudaGraph_t g = nullptr;
  CU(cudaStreamEndCapture(c->stream, &g));
  cudaGraphExec_t ge = nullptr;
  cudaError_t e = cudaGraphInstantiate(&ge, g, 0);
  cudaGraphDestroy(g);
  if (e != cudaSuccess) return fail(B200TFS_E_CUDA, "cudaGraphInstantiate: %s", cudaGetErrorString(e));
  c->has_graphs = true;
  *graph_exec = ge;
  return B200TFS_OK;
}

int b200tfs_graph_launch(b200tfs_ctx* c, void* graph_exec) {
  if (!c || !graph_exec) return fail(B200TFS_E_ARG, "NULL argument");
  CU(cudaGraphLaunch((cudaGraphExec_t)graph_exec, c->stream));
  return B200TFS_OK;
}

int b200tfs_graph_destroy(void* graph_exec) {
  if (graph_exec) CU(cudaGraphExecDestroy((cudaGraphExec_t)graph_exec));
  return B200TFS_OK;
}

int b200tfs_wait_event(b200tfs_ctx* c, void* ev) {
  if (!c || !ev) return fail(B200TFS_E_ARG, "NULL argument");
  CU(cudaStreamWaitEvent(c->stream, (cudaEvent_t)ev, 0));
  return B200TFS_OK;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------
// host-buffer entry points
// ------------------------------------------------------------------------------------------------
namespace {

// bytes of source memory a tensor occupies
uint64_t tensor_src_bytes(const b200tfs_tensor& t) {
  if (t.flags & B200TFS_F_PRESERIALIZED) return t.packed_len;
  uint64_t n = 1;
  for (int i = 0; i < t.rank; ++i) n *= (uint64_t)t.dims[i];
  return n * dtype_info(t.src_dtype).elem_size;
}

// one host tensor's place in the device staging buffer
struct StagePiece { const uint8_t* dev; const uint8_t* host; uint64_t nb; };

// Host-to-device copies of a batch, merged where consecutive ones continue each other on BOTH sides (a batch whose tensors lie
// back to back in one pinned buffer - bench.py's lanes, a caller's arena - becomes one copy instead of one per tensor: each copy
// costs driver time, a sizeable share of a 602 KB tensor's time on the link).
struct CopyMerger {
  cudaStream_t stream;
  uint8_t* d = nullptr; const uint8_t* h = nullptr; uint64_t n = 0;
  std::vector<std::pair<uint64_t, uint64_t>> parts;   // the copies merged into [d, d + n): offset from d (and h), bytes
  explicit CopyMerger(cudaStream_t s) : stream(s) {}
  cudaError_t add(const void* dst, const void* src, uint64_t nb) {
    if (!nb) return cudaSuccess;
    if (n && (const uint8_t*)dst >= d + n && (const uint8_t*)dst - (d + n) == (const uint8_t*)src - (h + n) && (const uint8_t*)dst - (d + n) < 256) {
      parts.push_back({(uint64_t)((const uint8_t*)dst - d), nb});
      n = (uint64_t)((const uint8_t*)dst - d) + nb;      // the gap (alignment padding, equal on both sides) travels along
      return cudaSuccess;
    }
    cudaError_t e = flush();
    d = (uint8_t*)dst; h = (const uint8_t*)src; n = nb;
    parts.assign(1, {0, nb});
    return e;
  }
  // Sources that lie at the staging gap from each other need not be one allocation: two page-locked buffers can sit that close,
  // and the runtime refuses a copy whose host range spans both (cudaErrorInvalidValue).  Such a range is copied part by part.
  cudaError_t flush() {
    cudaError_t e = cudaSuccess;
    if (n) e = cudaMemcpyAsync(d, h, n, cudaMemcpyHostToDevice, stream);
    if (e == cudaErrorInvalidValue && parts.size() > 1) {
      cudaGetLastError();
      e = cudaSuccess;
      for (size_t i = 0; i < parts.size() && e == cudaSuccess; ++i)
        e = cudaMemcpyAsync(d + parts[i].first, h + parts[i].first, parts[i].second, cudaMemcpyHostToDevice, stream);
    }
    n = 0;
    parts.clear();
    return e;
  }
};

// Give every tensor of the batch a place in the device staging buffer and return device-pointing clones.  `defer` == nullptr:
// the copies are queued on the context's stream right here; else they are only listed (the pipelined path issues them in slices).
int stage_tensors(b200tfs_ctx* c, std::vector<b200tfs_tensor>& ts, std::vector<StagePiece>* defer = nullptr) {
  uint64_t total = 0;
  for (auto& t : ts) {
    if (!(t.flags & B200TFS_F_PRESERIALIZED)) {
      if (dtype_info(t.src_dtype).kind == VK_NONE || dtype_info(t.src_dtype).kind == VK_STRING)
        return fail(B200TFS_E_DTYPE, "dtype %d has no device payload", t.src_dtype);
      if (t.rank < 0 || t.rank > 254 || (t.rank && !t.dims)) return fail(B200TFS_E_SHAPE, "bad rank/dims");
      for (int i = 0; i < t.rank; ++i) if (t.dims[i] < 0) return fail(B200TFS_E_SHAPE, "negative dim");
    }
    if (t.flags & B200TFS_F_DEVICE_DATA) continue;   // already in HBM
    total += tensor_src_bytes(t) + 255;      // whatever order the places are handed out in
  }
  int rc = grow_dev(c, c->stage_dev, total + 256);
  if (rc) return rc;
  // places are handed out in order of HOST address: tensors that lie back to back in the caller's memory (all images of a batch
  // in one buffer, all labels in another) then lie back to back in the staging buffer too, and their copies merge
  std::vector<uint32_t> order;
  order.reserve(ts.size());
  for (uint32_t i = 0; i < ts.size(); ++i) {
    if (ts[i].flags & B200TFS_F_DEVICE_DATA) { ts[i].flags &= ~B200TFS_F_DEVICE_DATA; continue; }
    order.push_back(i);
  }
  std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return (uintptr_t)ts[a].data < (uintptr_t)ts[b].data; });
  uint64_t cur = 0;
  CopyMerger cm(c->stream);
  for (uint32_t i : order) {
    b200tfs_tensor& t = ts[i];
    cur = (cur + 255) & ~255ull;
    uint64_t nb = tensor_src_bytes(t);
    if (nb) {
      if (!t.data) return fail(B200TFS_E_ARG, "tensor data pointer is NULL");
      if (defer) defer->push_back(StagePiece{(const uint8_t*)c->stage_dev.p + cur, (const uint8_t*)t.data, nb});
      else CU(cm.add((uint8_t*)c->stage_dev.p + cur, t.data, nb));
    }
    t.data = (uint8_t*)c->stage_dev.p + cur;
    cur += nb;
  }
  CU(cm.flush());
  return B200TFS_OK;
}

bool needs_measure_one(const b200tfs_tensor& t) {
  return !(t.flags & (B200TFS_F_PRESERIALIZED | B200TFS_F_TENSOR_CONTENT)) && dtype_info(t.wire_dtype).kind == VK_VARINT;
}
// a packed-varint input the host can measure itself: its values are in host memory, few, and well-formed
bool host_measurable_varint(const b200tfs_tensor& t) {
  if (!needs_measure_one(t) || t.src_dtype != t.wire_dtype || (t.flags & B200TFS_F_DEVICE_DATA)) return false;
  if (t.rank < 0 || t.rank > 254 || (t.rank && !t.dims)) return false;
  uint64_t ne = 1;
  for (int k = 0; k < t.rank; ++k) { if (t.dims[k] < 0 || t.dims[k] > 4096) return false; ne *= (uint64_t)t.dims[k]; if (ne > 4096) return false; }
  return ne == 0 || t.data != nullptr;
}

// Is this host pointer page-locked memory the device can address (cudaHostAlloc / cudaHostRegister under unified addressing)?
// Then a kernel may write its output there itself - posted PCIe writes at the link rate - and the device-to-host copy
// disappears.  (The other direction does not pay: SM-issued reads of host memory are slower than the copy engine's.)
uint8_t* device_view_of_host(const void* p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return nullptr; }
  if (a.type != cudaMemoryTypeHost || !a.devicePointer) return nullptr;
  return (uint8_t*)a.devicePointer;
}

// source bytes per output byte of a move op, as a fraction num/den; 0/0: the op cannot be cut
void op_ratio(uint32_t op, uint32_t* num, uint32_t* den) {
  switch (op) {
    case OP_COPY: case OP_QUIET_SRC: case OP_QUIET_DST: case OP_BOOL: *num = 1; *den = 1; break;
    case OP_H2F: case OP_B2F: *num = 1; *den = 2; break;
    case OP_F2H: case OP_F2B: *num = 2; *den = 1; break;
    default: *num = 0; *den = 0; break;
  }
}

// The pipelined encode: the batch's large payloads are cut into up to kPipeMax slices of consecutive wire bytes; slice k's source
// bytes travel H2D on one stream while slice k-1 is being encoded on the context's stream and slice k-2's wire bytes travel D2H on
// a third - one big request alone keeps both PCIe directions busy (VERDICT r1 weak #4: monolithic H2D -> kernel -> D2H).
// Framing bytes and small payloads go with slice 0.  Returns B200TFS_OK with *done = false when the batch does not qualify.
// `direct`: the plan's destinations already lie in the caller's (pinned) wire buffer: no device-to-host copies, two streams.
int encode_pipelined(b200tfs_ctx* c, PlanBuilder& pb, const std::vector<StagePiece>& pieces, uint8_t* wire_host, uint64_t lo, uint64_t hi,
                     bool direct, bool* done) {
  *done = false;
  if (!c->pipe_min || pb.large_bytes < c->pipe_min || !pb.varjobs.empty() || pb.items.empty()) return B200TFS_OK;
  for (auto& it : pb.items) {
    uint32_t num, den;
    op_ratio(it.op, &num, &den);
    if (!num || it.glen) return B200TFS_OK;
  }
  int K = (int)std::min<uint64_t>(c->pipe_max, std::max<uint64_t>(2, pb.large_bytes / std::max<uint64_t>(c->pipe_min, 1ull << 18)));
  const uint64_t per = ((pb.large_bytes + K - 1) / K + 65535) & ~65535ull;    // output bytes per slice, cut on 64 KB
  const uint8_t* arena = (const uint8_t*)c->arena_dev.p;
  // which piece feeds an item: the one that contains its source (device-resident inputs have none)
  auto piece_of = [&](const uint8_t* src) -> const StagePiece* {      // pieces are in ascending staging-address order (stage_tensors)
    auto it = std::upper_bound(pieces.begin(), pieces.end(), src, [](const uint8_t* s, const StagePiece& p) { return s < p.dev; });
    if (it == pieces.begin()) return nullptr;
    --it;
    return (src >= it->dev && src < it->dev + it->nb) ? &*it : nullptr;
  };
  std::vector<const StagePiece*> feeds(pb.items.size());
  std::vector<char> is_large(pieces.size(), 0);
  for (size_t i = 0; i < pb.items.size(); ++i) {
    feeds[i] = piece_of(pb.items[i].src);
    if (feeds[i]) is_large[feeds[i] - pieces.data()] = 1;
  }
  // everything queued on this context so far (the previous call's kernels read the staging buffer) precedes our copies
  cudaEvent_t* ev = c->pipe_ev;
  CU(cudaEventRecord(ev[2 * b200tfs_ctx::kPipeMax], c->stream));
  CU(cudaStreamWaitEvent(c->aux_stream, ev[2 * b200tfs_ctx::kPipeMax], 0));
  if (!direct) CU(cudaStreamWaitEvent(c->d2h_stream, ev[2 * b200tfs_ctx::kPipeMax], 0));
  size_t item = 0;
  uint64_t item_done = 0;        // output bytes of pb.items[item] already handed to a slice
  uint64_t wire_done = lo;       // arena offset up to which the wire has been copied back
  int rc;
  for (int k = 0; k < K && (item < pb.items.size() || k == 0); ++k) {
    PlanBuilder sub;
    CopyMerger cm(c->aux_stream);
    if (k == 0) {
      sub.smalls.swap(pb.smalls);
      sub.blob.swap(pb.blob);
      for (size_t q = 0; q < pieces.size(); ++q)     // sources of small payloads
        if (!is_large[q]) CU(cm.add(pieces[q].dev, pieces[q].host, pieces[q].nb));
      CU(cm.flush());
    }
    uint64_t room = per;
    uint64_t wire_end = wire_done;
    while (item < pb.items.size() && room) {
      const MoveItem& it = pb.items[item];
      uint32_t num, den;
      op_ratio(it.op, &num, &den);
      const bool last_slice = (k == K - 1);
      uint64_t take = std::min<uint64_t>(it.n_out - item_done, last_slice ? ~0ull : room);
      if (take < it.n_out - item_done) take &= ~1023ull;     // cuts fall on 1 KB of output: whole elements and whole 16-byte vectors of either side
      if (!take) break;
      if (!last_slice) room -= std::min(room, take);
      const uint64_t s_off = item_done * num / den, s_len = take * num / den;
      if (feeds[item]) CU(cm.add(it.src + s_off, feeds[item]->host + (it.src + s_off - feeds[item]->dev), s_len));
      sub.payload(it.src + s_off, it.dst + item_done, take, it.op);
      if (!direct) wire_end = (uint64_t)(it.dst + item_done + take - arena);
      item_done += take;
      if (item_done == it.n_out) { ++item; item_done = 0; }
    }
    const bool final_slice = item >= pb.items.size();
    if (final_slice) wire_end = hi;
    CU(cm.flush());
    CU(cudaEventRecord(ev[2 * k], c->aux_stream));
    CU(cudaStreamWaitEvent(c->stream, ev[2 * k], 0));
    if ((rc = launch_plan(c, sub))) return rc;
    if (!direct) {
      CU(cudaEventRecord(ev[2 * k + 1], c->stream));
      CU(cudaStreamWaitEvent(c->d2h_stream, ev[2 * k + 1], 0));
      if (wire_end > wire_done)
        CU(cudaMemcpyAsync(wire_host + (wire_done - lo), arena + wire_done, wire_end - wire_done, cudaMemcpyDeviceToHost, c->d2h_stream));
      wire_done = wire_end;
    }
    if (final_slice) break;
  }
  if (!direct) {   // the context's stream is where callers wait: it ends behind the last copy
    CU(cudaEventRecord(ev[2 * b200tfs_ctx::kPipeMax + 1], c->d2h_stream));
    CU(cudaStreamWaitEvent(c->stream, ev[2 * b200tfs_ctx::kPipeMax + 1], 0));
  }
  c->pipelined_calls += 1;
  *done = true;
  return B200TFS_OK;
}

}  // namespace

extern "C" {

int b200tfs_encode_tensor_protos_host(b200tfs_ctx* c, int32_t n, const b200tfs_tensor* tensors, void* wire_host, uint64_t wire_cap,
                                      uint64_t* rec_off, uint64_t* rec_len) {
  if (!c || n < 0 || (n && (!tensors || !wire_host || !rec_off || !rec_len))) return fail(B200TFS_E_ARG, "bad arguments");
  if (n == 0) return B200TFS_OK;
  CU(cudaSetDevice(c->device));
  std::vector<b200tfs_tensor> ts(tensors, tensors + n);
  int rc = stage_tensors(c, ts);
  if (rc) return rc;
  if ((rc = b200tfs_measure(c, n, ts.data()))) return rc;
  uint64_t need = 0;
  if ((rc = b200tfs_tensor_arena_size(n, ts.data(), &need))) return rc;
  if ((rc = grow_dev(c, c->arena_dev, need))) return rc;
  if ((rc = b200tfs_encode_tensor_protos(c, n, ts.data(), c->arena_dev.p, c->arena_dev.cap, rec_off, rec_len))) return rc;
  const uint64_t lo = rec_off[0], hi = rec_off[n - 1] + rec_len[n - 1];
  if (hi - lo > wire_cap) return fail(B200TFS_E_SIZE, "wire buffer too small: need %llu bytes", (unsigned long long)(hi - lo));
  CU(cudaMemcpyAsync(wire_host, (uint8_t*)c->arena_dev.p + lo, hi - lo, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  for (int i = 0; i < n; ++i) rec_off[i] -= lo;
  return B200TFS_OK;
}

static int encode_requests_host_async_spec(b200tfs_ctx* c, int32_t n, const b200tfs_request* reqs, const b200tfs_request_spec* specs,
                                           void* wire_host, uint64_t wire_cap, uint64_t* rec_off, uint64_t* rec_len) {
  if (!c || n < 0 || (n && (!reqs || !wire_host || !rec_off || !rec_len))) return fail(B200TFS_E_ARG, "bad arguments");
  if (n == 0) return B200TFS_OK;
  CU(cudaSetDevice(c->device));
  // flatten every input of every request, stage them, then rebuild request structs on the clones
  std::vector<b200tfs_tensor> ts;
  for (int i = 0; i < n; ++i) {
    if (reqs[i].n_inputs < 0 || (reqs[i].n_inputs && !reqs[i].inputs)) return fail(B200TFS_E_ARG, "bad request %d", i);
    ts.insert(ts.end(), reqs[i].inputs, reqs[i].inputs + reqs[i].n_inputs);
  }
  // Packed-varint inputs of up to 4096 elements that lie in HOST memory (labels, ids, one sequence of token ids) are measured
  // right here - a few microseconds of host arithmetic instead of a counting kernel, a device-to-host copy and a stream
  // synchronise (b200tfs_measure: the call can queue nothing else until that round trip is over).
  bool device_measure = false;
  for (auto& t : ts) {
    if (!host_measurable_varint(t)) { device_measure = device_measure || needs_measure_one(t); continue; }
    uint64_t ne = 1;
    for (int k = 0; k < t.rank; ++k) ne *= (uint64_t)t.dims[k];
    const DtypeInfo di = dtype_info(t.src_dtype);
    t.packed_len = ne ? tiny_total(TinyVar{(const uint8_t*)t.data, (uint32_t)ne, di.elem_size, di.is_signed, 0}) : 0;
  }
  // a batch that needs no device measuring may take the pipelined path: its H2D copies are then issued slice by slice
  const bool try_pipe = c->pipe_min && !c->capturing && !device_measure;
  std::vector<StagePiece> pieces;
  int rc = stage_tensors(c, ts, try_pipe ? &pieces : nullptr);
  if (rc) return rc;
  if (device_measure && (rc = b200tfs_measure(c, (int32_t)ts.size(), ts.data()))) return rc;  // synchronises
  std::vector<b200tfs_request> rq(reqs, reqs + n);
  size_t k = 0;
  for (int i = 0; i < n; ++i) { rq[i].inputs = ts.data() + k; k += (size_t)rq[i].n_inputs; }
  uint64_t need = 0;
  if ((rc = b200tfs_request_arena_size_spec(n, rq.data(), specs, &need))) return rc;
  if (try_pipe) {
    // A pinned wire buffer with room for the arena layout (records 256-byte aligned, largest payload 128-byte aligned) is written
    // by the kernels themselves; rec_off then counts from wire_host like always, but record 0 does not start at 0.
    uint8_t* out_dev = (c->opt_direct_out && c->pipe_min && need <= wire_cap) ? device_view_of_host(wire_host) : nullptr;
    if (out_dev && ((uintptr_t)out_dev & 255)) out_dev = nullptr;
    const bool direct = out_dev != nullptr;
    if (!direct && (rc = grow_dev(c, c->arena_dev, need))) return rc;
    PlanBuilder pb;
    if ((rc = plan_requests(n, rq.data(), specs, direct ? (void*)out_dev : c->arena_dev.p, direct ? wire_cap : c->arena_dev.cap, rec_off, rec_len,
                            pb)))
      return rc;
    const uint64_t lo = rec_off[0], hi = rec_off[n - 1] + rec_len[n - 1];
    if (!direct && hi - lo > wire_cap) return fail(B200TFS_E_SIZE, "wire buffer too small: need %llu bytes", (unsigned long long)(hi - lo));
    bool done = false;
    if ((rc = encode_pipelined(c, pb, pieces, (uint8_t*)wire_host, lo, hi, direct, &done))) return rc;
    if (!done) {   // too small to be worth slicing: everything on the context's stream, as one piece
      CopyMerger cm(c->stream);
      for (auto& p : pieces) CU(cm.add(p.dev, p.host, p.nb));
      CU(cm.flush());
      if ((rc = launch_plan(c, pb))) return rc;
      if ((rc = run_varjobs(c, pb))) return rc;
      if (!direct) CU(cudaMemcpyAsync(wire_host, (uint8_t*)c->arena_dev.p + lo, hi - lo, cudaMemcpyDeviceToHost, c->stream));
    }
    if (direct) c->direct_calls += 1;
    else for (int i = 0; i < n; ++i) rec_off[i] -= lo;
    return B200TFS_OK;
  }
  if ((rc = grow_dev(c, c->arena_dev, need))) return rc;
  if ((rc = encode_requests_spec(c, n, rq.data(), specs, c->arena_dev.p, c->arena_dev.cap, rec_off, rec_len))) return rc;
  const uint64_t lo = rec_off[0], hi = rec_off[n - 1] + rec_len[n - 1];
  if (hi - lo > wire_cap) return fail(B200TFS_E_SIZE, "wire buffer too small: need %llu bytes", (unsigned long long)(hi - lo));
  CU(cudaMemcpyAsync(wire_host, (uint8_t*)c->arena_dev.p + lo, hi - lo, cudaMemcpyDeviceToHost, c->stream));
  for (int i = 0; i < n; ++i) rec_off[i] -= lo;
  return B200TFS_OK;
}

int b200tfs_encode_requests_host_async(b200tfs_ctx* c, int32_t n, const b200tfs_request* reqs, void* wire_host, uint64_t wire_cap,
                                       uint64_t* rec_off, uint64_t* rec_len) {
  return encode_requests_host_async_spec(c, n, reqs, nullptr, wire_host, wire_cap, rec_off, rec_len);
}

int b200tfs_pipelined_calls(b200tfs_ctx* c, uint64_t* count) {
  if (!c || !count) return fail(B200TFS_E_ARG, "bad arguments");
  *count = c->pipelined_calls;
  return B200TFS_OK;
}

int b200tfs_direct_calls(b200tfs_ctx* c, uint64_t* count) {
  if (!c || !count) return fail(B200TFS_E_ARG, "bad arguments");
  *count = c->direct_calls;
  return B200TFS_OK;
}

int b200tfs_set_pipeline(b200tfs_ctx* c, uint64_t min_bytes, int32_t max_slices) {
  if (!c) return fail(B200TFS_E_ARG, "ctx is NULL");
  if (min_bytes && (max_slices < 2 || max_slices > b200tfs_ctx::kPipeMax)) return fail(B200TFS_E_ARG, "max_slices must be in [2, %d]", b200tfs_ctx::kPipeMax);
  c->pipe_min = min_bytes;
  if (min_bytes) c->pipe_max = max_slices;
  return B200TFS_OK;
}

int b200tfs_encode_requests_host(b200tfs_ctx* c, int32_t n, const b200tfs_request* reqs, void* wire_host, uint64_t wire_cap,
                                 uint64_t* rec_off, uint64_t* rec_len) {
  return b200tfs_encode_requests_host_spec(c, n, reqs, nullptr, wire_host, wire_cap, rec_off, rec_len);
}

int b200tfs_encode_requests_host_spec(b200tfs_ctx* c, int32_t n, const b200tfs_request* reqs, const b200tfs_request_spec* specs,
                                      void* wire_host, uint64_t wire_cap, uint64_t* rec_off, uint64_t* rec_len) {
  int rc = encode_requests_host_async_spec(c, n, reqs, specs, wire_host, wire_cap, rec_off, rec_len);
  if (rc) return rc;
  CU(cudaStreamSynchronize(c->stream));
  return B200TFS_OK;
}

// Give a host wire its place in stage_dev, `shift` bytes in, and copy it there unless `copy` is false (the caller copies it in
// pieces).  *span receives the bytes the records cover.
static int stage_wire(b200tfs_ctx* c, const void* wire_host, int32_t n, const uint64_t* rec_off, const uint64_t* rec_len, uint64_t* span,
                      uint64_t shift = 0, bool copy = true) {
  uint64_t hi = 0;
  for (int i = 0; i < n; ++i) hi = std::max(hi, rec_off[i] + rec_len[i]);
  int rc = grow_dev(c, c->stage_dev, hi + 64);
  if (rc) return rc;
  c->stage_shift = shift;
  if (hi && copy) CU(cudaMemcpyAsync((uint8_t*)c->stage_dev.p + shift, wire_host, hi, cudaMemcpyHostToDevice, c->stream));
  *span = hi;
  return B200TFS_OK;
}

int b200tfs_parse_responses_host(b200tfs_ctx* c, const void* wire_host, int32_t n, const uint64_t* rec_off, const uint64_t* rec_len,
                                 int32_t max_outputs, b200tfs_output* outs, int32_t* n_outs, b200tfs_model_spec* specs,
                                 int32_t* rec_status) {
  if (!c || n < 0 || (n && (!wire_host || !rec_off || !rec_len))) return fail(B200TFS_E_ARG, "bad arguments");
  if (n == 0) return B200TFS_OK;
  CU(cudaSetDevice(c->device));
  uint64_t span;
  int rc = stage_wire(c, wire_host, n, rec_off, rec_len, &span);
  if (rc) return rc;
  return parse_common(c, c->stage_dev.p, n, rec_off, rec_len, max_outputs, false, outs, n_outs, specs, rec_status);
}

int b200tfs_parse_tensor_protos_host(b200tfs_ctx* c, const void* wire_host, int32_t n, const uint64_t* rec_off, const uint64_t* rec_len,
                                     b200tfs_output* outs, int32_t* rec_status) {
  if (!c || n < 0 || (n && (!wire_host || !rec_off || !rec_len))) return fail(B200TFS_E_ARG, "bad arguments");
  if (n == 0) return B200TFS_OK;
  CU(cudaSetDevice(c->device));
  uint64_t span;
  int rc = stage_wire(c, wire_host, n, rec_off, rec_len, &span);
  if (rc) return rc;
  return parse_common(c, c->stage_dev.p, n, rec_off, rec_len, 1, true, outs, nullptr, nullptr, rec_status);
}

int b200tfs_decode_responses_host_async(b200tfs_ctx* c, const void* wire_host, int32_t n, const uint64_t* rec_off, const uint64_t* rec_len,
                                        void* dst_host, uint64_t dst_stride) {
  if (!c || n < 0 || (n && (!wire_host || !rec_off || !rec_len || !dst_host))) return fail(B200TFS_E_ARG, "bad arguments");
  if (n == 0) return B200TFS_OK;
  if (dst_stride & 255) return fail(B200TFS_E_ARG, "dst_stride must be a multiple of 256");
  CU(cudaSetDevice(c->device));
  // The wire is in host memory: walk record 0 HERE (sub-microsecond: the walk steps over the payload) so that the launch
  // takes the template path from its first CTA on, and place the copy so that the largest value chunk lands 16-byte
  // aligned on the device (aligned loads and stores, no funnel shifts).
  const uint32_t vpt = decode_vpt(c, n, rec_len);
  Template T;
  uint64_t shift = 0;
  const bool have = vpt <= kStageVecsHost && !c->capturing &&
                    host_template((const uint8_t*)wire_host + rec_off[0], rec_len[0], vpt, dst_stride, c->serial + 1 ? c->serial + 1 : 1, c->decode_cast,
                                  c->decode_varints, &T);
  if (have) {
    uint32_t big = 0;
    for (uint32_t q = 1; q < T.in.head.n_chunks; ++q) if (T.in.chunk[q].len > T.in.chunk[big].len) big = q;
    if (T.in.head.n_chunks) shift = (16 - ((rec_off[0] + T.in.chunk[big].wire_off) & 15)) & 15;
  }
  // One large record whose values lie in one fixed-width chunk: slices of tiles, pipelined like the encode (wire bytes of slice
  // k+1 travel H2D while slice k is decoded and the tensor bytes of slice k-1 travel D2H).  The kernel skips its framing verdict:
  // the template was built from these very bytes, and a slice runs before the record's tail has arrived.
  const TplChunk& ch = T.in.chunk[0];
  const uint64_t tile_bytes = 16ull * vpt;
  const bool sliced = have && n == 1 && c->pipe_min && rec_len[0] >= c->pipe_min && !c->opt_no_inline && T.in.head.n_chunks == 1 &&
                      !ch.is_varint && (ch.op == OP_COPY || ch.op == OP_QUIET_DST) && ch.n_tiles >= 2 && ch.n_tiles == T.in.head.total_tiles;
  uint64_t hi;
  int rc = stage_wire(c, wire_host, n, rec_off, rec_len, &hi, shift, !sliced);
  if (rc) return rc;
  // a pinned destination is written by the kernel itself (posted PCIe writes): no staging buffer, no device-to-host copy
  uint8_t* dst_direct = (c->opt_direct_out && c->pipe_min) ? device_view_of_host(dst_host) : nullptr;
  if (dst_direct && ((uintptr_t)dst_direct & 255)) dst_direct = nullptr;
  if (!dst_direct && (rc = grow_dev(c, c->arena_dev, dst_stride * (uint64_t)n + 256))) return rc;
  uint8_t* dst_dev = dst_direct ? dst_direct : (uint8_t*)c->arena_dev.p;
  if (dst_direct) c->direct_calls += 1;
  uint8_t* wire_dev = (uint8_t*)c->stage_dev.p + shift;
  if (sliced) {
    DecodeSlices sl;
    sl.K = (int)std::min<uint64_t>(std::min<uint64_t>(c->pipe_max, ch.n_tiles),
                                   std::max<uint64_t>(2, rec_len[0] / std::max<uint64_t>(c->pipe_min, 1ull << 18)));
    for (int k = 0; k <= sl.K; ++k) sl.tile_lo[k] = (uint32_t)((uint64_t)ch.n_tiles * k / sl.K);
    cudaEvent_t* ev = c->pipe_ev;
    sl.before = ev; sl.after = ev + b200tfs_ctx::kPipeMax;
    CU(cudaEventRecord(ev[2 * b200tfs_ctx::kPipeMax], c->stream));
    CU(cudaStreamWaitEvent(c->aux_stream, ev[2 * b200tfs_ctx::kPipeMax], 0));
    if (!dst_direct) CU(cudaStreamWaitEvent(c->d2h_stream, ev[2 * b200tfs_ctx::kPipeMax], 0));
    uint64_t wire_done = 0;
    for (int k = 0; k < sl.K; ++k) {
      // tiles below tile_lo[k+1] read no further than 48 bytes past their last vector (the next 16-byte block of a shifted source)
      const uint64_t w_end = (k + 1 == sl.K) ? hi : std::min<uint64_t>(hi, rec_off[0] + ch.wire_off + sl.tile_lo[k + 1] * tile_bytes + 64);
      if (w_end > wire_done)
        CU(cudaMemcpyAsync(wire_dev + wire_done, (const uint8_t*)wire_host + wire_done, w_end - wire_done, cudaMemcpyHostToDevice, c->aux_stream));
      wire_done = std::max(wire_done, w_end);
      CU(cudaEventRecord(sl.before[k], c->aux_stream));
    }
    if ((rc = decode_launch(c, wire_dev, n, rec_off, rec_len, dst_dev, dst_stride, vpt, &T, &sl))) return rc;
    if (!dst_direct) {
      const uint64_t need = std::min<uint64_t>(dst_stride, T.in.head.dst_need);
      uint64_t dst_done = 0;
      for (int k = 0; k < sl.K; ++k) {
        // tiles below tile_lo[k+1] have written every byte of the slot below the first vector of tile tile_lo[k+1]
        const uint64_t d_end = (k + 1 == sl.K) ? need : std::min<uint64_t>(need, ch.dst_off + sl.tile_lo[k + 1] * tile_bytes);
        CU(cudaStreamWaitEvent(c->d2h_stream, sl.after[k], 0));
        if (d_end > dst_done)
          CU(cudaMemcpyAsync((uint8_t*)dst_host + dst_done, (uint8_t*)c->arena_dev.p + dst_done, d_end - dst_done, cudaMemcpyDeviceToHost, c->d2h_stream));
        dst_done = std::max(dst_done, d_end);
      }
      CU(cudaEventRecord(ev[2 * b200tfs_ctx::kPipeMax + 1], c->d2h_stream));
      CU(cudaStreamWaitEvent(c->stream, ev[2 * b200tfs_ctx::kPipeMax + 1], 0));
    }
    c->pipelined_calls += 1;
    return B200TFS_OK;
  }
  if ((rc = decode_launch(c, wire_dev, n, rec_off, rec_len, dst_dev, dst_stride, vpt, have ? &T : nullptr))) return rc;
  if (!dst_direct) CU(cudaMemcpyAsync(dst_host, c->arena_dev.p, dst_stride * (uint64_t)n, cudaMemcpyDeviceToHost, c->stream));
  return B200TFS_OK;
}

int b200tfs_unpack_outputs_host(b200tfs_ctx* c, int32_t m, const b200tfs_output* outs, const uint64_t* out_rec_off, void* const* dst_host,
                                const int32_t* dst_dtype, int32_t* status) {
  if (!c || m < 0 || (m && (!outs || !dst_host))) return fail(B200TFS_E_ARG, "bad arguments");
  if (m == 0) return B200TFS_OK;
  CU(cudaSetDevice(c->device));
  if (!c->stage_dev.p) return fail(B200TFS_E_ARG, "no staged wire: call b200tfs_parse_*_host first");
  std::vector<uint64_t> off(m), nb(m);
  uint64_t total = 0;
  for (int j = 0; j < m; ++j) {
    int32_t want = dst_dtype ? dst_dtype[j] : outs[j].dtype;
    if (want == B200TFS_DT_HALF_REFQUIRK) want = DT_HALF;
    nb[j] = outs[j].n_elems * dtype_info(want).elem_size;
    total = (total + 255) & ~255ull;
    off[j] = total;
    total += nb[j];
  }
  int rc = grow_dev(c, c->arena_dev, total + 256);
  if (rc) return rc;
  std::vector<void*> dd(m);
  for (int j = 0; j < m; ++j) dd[j] = (uint8_t*)c->arena_dev.p + off[j];
  if ((rc = unpack_outputs_impl(c, (uint8_t*)c->stage_dev.p + c->stage_shift, m, outs, out_rec_off, dd.data(), dst_dtype, status, false))) return rc;
  for (int j = 0; j < m; ++j)
    if (nb[j]) {
      if (!dst_host[j]) return fail(B200TFS_E_ARG, "output %d: dst is NULL", j);
      CU(cudaMemcpyAsync(dst_host[j], dd[j], nb[j], cudaMemcpyDeviceToHost, c->stream));
    }
  CU(cudaStreamSynchronize(c->stream));
  collect_varint_status(c, status);
  return B200TFS_OK;
}

// ------------------------------------------------------------------------------------------------
// decode into one tensor per key, concatenated along axis 0
// ------------------------------------------------------------------------------------------------
extern "C++" {
template <class Key>   // b200tfs_concat_key, b200tfs_pad_key
static int concat_check_keys(int32_t n_keys, const Key* keys) {
  if (n_keys <= 0 || n_keys > B200TFS_CONCAT_MAX_KEYS || !keys) return fail(B200TFS_E_ARG, "n_keys must be 1..%d", B200TFS_CONCAT_MAX_KEYS);
  for (int k = 0; k < n_keys; ++k) {
    if (keys[k].key_len < 0 || keys[k].key_len > 0xFFFFFFFFll || (keys[k].key_len && !keys[k].key)) return fail(B200TFS_E_ARG, "key %d: bad key", k);
    for (int j = 0; j < k; ++j)
      if (keys[j].key_len == keys[k].key_len && !memcmp(keys[j].key, keys[k].key, (size_t)keys[k].key_len))
        return fail(B200TFS_E_ARG, "key %d repeats key %d", k, j);
  }
  return B200TFS_OK;
}
}  // extern "C++"

int b200tfs_response_keys(const void* rec_host, uint64_t rec_len, int32_t cap, uint64_t* key_off, uint32_t* key_len, int32_t* count) {
  if (!count || cap < 0 || (cap && (!key_off || !key_len)) || (rec_len && !rec_host)) return fail(B200TFS_E_ARG, "bad arguments");
  *count = 0;
  std::vector<b200tfs_output> outs;
  for (int max = 16;; max *= 2) {   // PredictResponse.FromString has no limit on the map size
    outs.assign((size_t)max + 1, b200tfs_output{});
    b200tfs_model_spec spec;
    int cnt = 0;
    std::vector<SpillEntry> spill(4096);
    const int st = walk_host_record(rec_host, rec_len, max, outs.data(), &cnt, &spec, SpillArea{spill.data(), (uint32_t)spill.size(), 0u});
    if (st == B200TFS_E_SIZE && max < (1 << 20)) continue;
    if (st != B200TFS_OK && st != B200TFS_E_SPILL) return st;   // a spill only concerns dims / runs: the keys are all there
    *count = cnt;
    for (int i = 0; i < cnt && i < cap; ++i) { key_off[i] = outs[i].key_off; key_len[i] = outs[i].key_len; }
    return B200TFS_OK;
  }
}

extern "C++" {
// The host walk of b200tfs_concat_layout and b200tfs_padded_layout: per key, the first problem in record order, the dtype and
// rank of the first record that has the key, the rows, and the trailing dims - every record's (another one is E_SHAPE) or, with
// `ragged`, their elementwise maximum.  `on_out(k, record, its length, output)` sees every output that passes those checks and
// may refuse it with a status.
template <class Key, class OnOut>
static int key_layout(const void* wire_host, int32_t n, const uint64_t* rec_off, const uint64_t* rec_len, int32_t n_keys, Key* keys,
                      int32_t cast, bool ragged, OnOut&& on_out) {
  if (n <= 0 || !wire_host || !rec_off || !rec_len) return fail(B200TFS_E_ARG, "bad arguments");
  int rc = concat_check_keys(n_keys, keys);
  if (rc) return rc;
  if (cast != 0 && cast != DT_FLOAT && cast != DT_HALF && cast != DT_BFLOAT16) return fail(B200TFS_E_DTYPE, "cast to dtype %d", cast);
  const uint32_t cst = (cast == DT_HALF || cast == DT_BFLOAT16) ? (uint32_t)cast : 0u;
  for (int k = 0; k < n_keys; ++k) {
    Key& K = keys[k];
    K.dtype = 0; K.rank = 0; K.bytes = 0; K.status = B200TFS_E_KEY; K.bad_rec = -1;
    for (int d = 0; d < B200TFS_MAX_RANK; ++d) K.dims[d] = 0;
  }
  std::vector<uint8_t> have(n_keys, 0);   // a reference record for the key was found
  std::vector<int> done(n_keys, 0);       // the key's status is final
  for (int r = 0; r < n; ++r) {
    b200tfs_output outs[kFusedMaxOutputs + 1];
    b200tfs_model_spec spec;
    int cnt = 0;
    const uint8_t* rec = (const uint8_t*)wire_host + rec_off[r];
    int st = walk_host_record(rec, rec_len[r], kFusedMaxOutputs, outs, &cnt, &spec);
    if (st == B200TFS_E_SPILL || st == B200TFS_E_SIZE) st = B200TFS_E_NONCANONICAL;
    for (int k = 0; k < n_keys; ++k) {
      if (done[k]) continue;
      Key& K = keys[k];
      int32_t s = st;
      const b200tfs_output* o = nullptr;
      if (s == B200TFS_OK) {
        for (int j = 0; j < cnt && !o; ++j)
          if ((int64_t)outs[j].key_len == K.key_len && !memcmp(rec + outs[j].key_off, K.key, (size_t)K.key_len)) o = &outs[j];
        if (!o) s = B200TFS_E_KEY;
        else if ((s = o->status) == B200TFS_OK) {
          if (o->rank == 0) s = B200TFS_E_SHAPE;
          else if (o->rank > B200TFS_MAX_RANK) s = B200TFS_E_NONCANONICAL;
          else if (have[k] && o->dtype != K.dtype) s = B200TFS_E_DTYPE;
          else if (have[k] && o->rank != K.rank) s = B200TFS_E_SHAPE;
          else for (int d = 1; have[k] && !ragged && d < o->rank; ++d) if (o->dims[d] != K.dims[d]) s = B200TFS_E_SHAPE;
          if (s == B200TFS_OK) s = on_out(k, rec, rec_len[r], *o);
        }
      }
      if (s != B200TFS_OK) { K.status = s; K.bad_rec = r; done[k] = 1; continue; }
      if (!have[k]) {
        have[k] = 1;
        K.dtype = o->dtype; K.rank = o->rank;
        for (int d = 0; d < o->rank; ++d) K.dims[d] = o->dims[d];
        K.dims[0] = 0;
      }
      K.dims[0] += o->dims[0];
      for (int d = 1; ragged && d < o->rank; ++d) K.dims[d] = std::max(K.dims[d], o->dims[d]);
      if (!ragged) K.bytes += tpl_narrows(cst, o->dtype) ? o->n_elems * 2 : o->dst_bytes;
    }
  }
  for (int k = 0; k < n_keys; ++k) {
    Key& K = keys[k];
    if (!done[k]) K.status = B200TFS_OK;
    if (ragged && K.status == B200TFS_OK) {
      uint64_t b = (uint64_t)K.dims[0] * (tpl_narrows(cst, K.dtype) ? 2u : dtype_info(K.dtype).elem_size);
      for (int d = 1; d < K.rank; ++d) b *= (uint64_t)K.dims[d];
      K.bytes = b;
    }
  }
  return B200TFS_OK;
}
}  // extern "C++"

int b200tfs_concat_layout(const void* wire_host, int32_t n, const uint64_t* rec_off, const uint64_t* rec_len, int32_t n_keys,
                          b200tfs_concat_key* keys, int32_t cast) {
  return b200tfs_concat_strings_layout(wire_host, n, rec_off, rec_len, n_keys, keys, nullptr, cast);
}

namespace {
struct StrTally {
  uint64_t bytes = 0;
  void operator()(uint64_t, uint32_t, uint32_t len) { bytes += len; }
};

// the walk of the index kernels over DT_STRING output o of a record: the strings of the entry's last `value` occurrence, added to
// *strings and *bytes, or B200TFS_E_NONCANONICAL when that is not all of them
int32_t tally_strings(const uint8_t* rec, uint64_t len, const b200tfs_output& o, uint64_t* strings, uint64_t* bytes) {
  Cursor c;
  cur_open_host(c, rec, (uint32_t)len);
  c.p = (uint32_t)o.msg_off;
  c.end = (uint32_t)(o.msg_off + o.msg_len);
  StrTally t;
  const uint64_t found = walk_strings(c, t);
  if (c.err || found != o.n_strings) return B200TFS_E_NONCANONICAL;
  *strings += found;
  *bytes += t.bytes;
  return B200TFS_OK;
}
}  // namespace

int b200tfs_concat_strings_layout(const void* wire_host, int32_t n, const uint64_t* rec_off, const uint64_t* rec_len, int32_t n_keys,
                                  b200tfs_concat_key* keys, b200tfs_concat_strings* strings, int32_t cast) {
  if (strings && n_keys > 0 && n_keys <= B200TFS_CONCAT_MAX_KEYS)
    for (int k = 0; k < n_keys; ++k) strings[k].strings = strings[k].data_bytes = 0;
  const int rc = key_layout(wire_host, n, rec_off, rec_len, n_keys, keys, cast, false,
                            [&](int k, const uint8_t* rec, uint64_t len, const b200tfs_output& o) -> int32_t {
                              if (!strings || dtype_info(o.dtype).kind != VK_STRING) return B200TFS_OK;
                              return tally_strings(rec, len, o, &strings[k].strings, &strings[k].data_bytes);
                            });
  if (rc || !strings) return rc;
  for (int k = 0; k < n_keys; ++k) {
    if (keys[k].status == B200TFS_OK && dtype_info(keys[k].dtype).kind == VK_STRING) keys[k].bytes = 8 * (strings[k].strings + 1);
    else strings[k].strings = strings[k].data_bytes = 0;
  }
  return B200TFS_OK;
}

int b200tfs_concat_strings_bound(int32_t n, const uint64_t* rec_len, uint64_t* max_strings, uint64_t* max_data_bytes) {
  if (n < 0 || (n && !rec_len)) return fail(B200TFS_E_ARG, "bad arguments");
  uint64_t s = 0, b = 0;
  for (int i = 0; i < n; ++i) { s += str_count_bound(rec_len[i]); b += rec_len[i]; }
  if (max_strings) *max_strings = s;
  if (max_data_bytes) *max_data_bytes = b;
  return B200TFS_OK;
}

int b200tfs_padded_layout(const void* wire_host, int32_t n, const uint64_t* rec_off, const uint64_t* rec_len, int32_t n_keys,
                          b200tfs_pad_key* keys, int32_t cast) {
  return b200tfs_padded_strings_layout(wire_host, n, rec_off, rec_len, n_keys, keys, nullptr, cast);
}

int b200tfs_padded_strings_layout(const void* wire_host, int32_t n, const uint64_t* rec_off, const uint64_t* rec_len, int32_t n_keys,
                                  b200tfs_pad_key* keys, b200tfs_padded_strings* strings, int32_t cast) {
  if (strings && n_keys > 0 && n_keys <= B200TFS_CONCAT_MAX_KEYS)
    for (int k = 0; k < n_keys; ++k) strings[k].strings = strings[k].data_bytes = 0;
  const int rc = key_layout(wire_host, n, rec_off, rec_len, n_keys, keys, cast, true,
                            [&](int k, const uint8_t* rec, uint64_t len, const b200tfs_output& o) -> int32_t {
                              if (!strings || dtype_info(o.dtype).kind != VK_STRING) return B200TFS_OK;
                              return tally_strings(rec, len, o, &strings[k].strings, &strings[k].data_bytes);
                            });
  if (rc || !strings) return rc;
  for (int k = 0; k < n_keys; ++k) {
    b200tfs_pad_key& K = keys[k];
    if (K.status == B200TFS_OK && dtype_info(K.dtype).kind == VK_STRING) {
      uint64_t m = (uint64_t)K.dims[0];
      for (int d = 1; d < K.rank; ++d) m *= (uint64_t)K.dims[d];
      K.bytes = 8 * (m + 1);
    } else {
      strings[k].strings = strings[k].data_bytes = 0;
    }
  }
  return B200TFS_OK;
}

namespace {
// device scratch of a per-key decode (b200tfs_decode_concat, b200tfs_decode_padded) for n records, n_keys keys and var_tile_cap
// varint tiles: the parse table, the keys' verdicts and matches, the varint tail's table and scratch, then the route's own
// regions of `sizes` bytes (own[i])
struct KeyLayout { uint64_t outs, nouts, specs, status, spill, kst, match, vouts, vnouts, vstatus, var, var_status, own[4], bytes; };
KeyLayout key_scratch(uint64_t n, uint64_t n_keys, uint64_t var_tile_cap, std::initializer_list<uint64_t> sizes) {
  const VarPlanLayout V = var_plan_layout(n, var_tile_cap);
  Layout R;
  KeyLayout L{};
  L.outs = R.take(sizeof(b200tfs_output) * n * (kFusedMaxOutputs + 1), 256);
  L.nouts = R.take(4 * n, 256);
  L.specs = R.take(sizeof(b200tfs_model_spec) * n, 256);
  L.status = R.take(4 * n, 256);
  L.spill = R.take(4 * n, 256);
  L.kst = R.take(4 * n * n_keys, 256);
  L.match = R.take(4 * n * n_keys, 256);
  L.vouts = R.take(sizeof(b200tfs_output) * n * kFusedMaxOutputs, 256);
  L.vnouts = R.take(4 * n, 256);
  L.vstatus = R.take(4 * n, 256);
  L.var = R.take(V.bytes, 256);
  L.var_status = L.var + V.status;
  uint64_t* own = L.own;
  for (uint64_t b : sizes) *own++ = R.take(b, 256);
  L.bytes = R.end;
  return L;
}
}  // namespace

extern "C++" {
// The start of a per-key decode: the argument checks (`check(key, k)`: the route's own checks of key k, after the shared ones),
// the device, and the varint tail's tile bound
template <class Key, class Check>
static int key_begin(b200tfs_ctx* c, const void* arena_dev, int32_t n, const uint64_t* rec_off, const uint64_t* rec_len, int32_t n_keys,
                     const Key* keys, uint64_t* var_tile_cap, Check&& check) {
  if (!c || n <= 0 || !arena_dev || !rec_off || !rec_len) return fail(B200TFS_E_ARG, "bad arguments");
  int rc = concat_check_keys(n_keys, keys);
  if (rc) return rc;
  for (int k = 0; k < n_keys; ++k) {
    if (keys[k].dst_cap && !keys[k].dst) return fail(B200TFS_E_ARG, "key %d: dst is NULL", k);
    if ((rc = check(keys[k], k))) return rc;
  }
  if (!c->capturing) CU(cudaSetDevice(c->device));
  uint64_t tiles = 0;
  for (int i = 0; i < n; ++i) tiles += var_record_tile_bound(rec_len[i]);
  if (tiles > 0x7FFFFFFFull) return fail(B200TFS_E_TOOBIG, "batch needs more than 2^31 tiles");
  *var_tile_cap = tiles;
  return B200TFS_OK;
}

// A per-key decode on c->stream, around the route's plan: its scratch in `g` (KeyLayout, with the route's regions `own`), one
// upload of rec_off | rec_len | key records (`dev_key(key, its bytes on the device)`) | key bytes, the parse kernel and the
// ConcatPlan fields both routes use.  `plan(cp, scratch, layout, device key records, device rec_len, &pad)` launches the route's kernels, which
// write the single-launch decode's table with absolute dst_off, and may set `pad`, the placement of the varint emit.  Then the
// varint tail over that table, and `res` becomes this call's.
// `extra`: n_extra more host byte ranges (the padded string decode's pad strings), uploaded behind the key bytes; extra[i].dev
// receives where range i lies on the device before `plan` runs.
struct HostBytes { const void* p; uint64_t len; const uint8_t* dev; };
template <class Key, class DevKey, class Plan>
static int key_decode(b200tfs_ctx* c, Growable& g, b200tfs_ctx::KeyResults& res, const void* arena_dev, int32_t n, const uint64_t* rec_off,
                      const uint64_t* rec_len, int32_t n_keys, const Key* keys, uint64_t var_tile_cap, std::initializer_list<uint64_t> own,
                      DevKey&& dev_key, Plan&& plan, HostBytes* extra = nullptr, int n_extra = 0) {
  using KeyRec = decltype(dev_key(keys[0], (const uint8_t*)nullptr));
  const KeyLayout L = key_scratch((uint64_t)n, (uint64_t)n_keys, var_tile_cap, own);
  int rc = grow_dev(c, g, L.bytes);
  if (rc) return rc;
  // rec_off | rec_len | keys | key bytes | extra: one upload (a captured call keeps a private copy)
  uint64_t key_bytes = 0;
  for (int k = 0; k < n_keys; ++k) key_bytes += (uint64_t)keys[k].key_len;
  for (int i = 0; i < n_extra; ++i) key_bytes += extra[i].len;
  Layout K;
  const uint64_t o_off = K.take(8ull * n), o_len = K.take(8ull * n), o_keys = K.take(sizeof(KeyRec) * n_keys), o_kb = K.take(key_bytes);
  Slot* slot;
  uint8_t* sd;
  rc = upload_image(c, K.end, {{o_off, rec_off, 8ull * n}, {o_len, rec_len, 8ull * n}}, &sd, &slot, [&](uint8_t* h, uint8_t* dev) {
    uint64_t at = o_kb;
    for (int k = 0; k < n_keys; ++k) {
      const KeyRec kd = dev_key(keys[k], dev + at);
      memcpy(h + o_keys + sizeof(KeyRec) * k, &kd, sizeof kd);
      if (keys[k].key_len) memcpy(h + at, keys[k].key, (size_t)keys[k].key_len);
      at += (uint64_t)keys[k].key_len;
    }
    for (int i = 0; i < n_extra; ++i) {
      if (extra[i].len) memcpy(h + at, extra[i].p, (size_t)extra[i].len);
      extra[i].dev = dev + at;
      at += extra[i].len;
    }
  });
  if (rc) return rc;
  for (int k = 0; k < n_keys; ++k) res.dst[k] = (uint8_t*)keys[k].dst;
  uint8_t* d = (uint8_t*)g.p;
  const uint64_t* off_dev = (const uint64_t*)(sd + o_off);
  CU(launch_parse_responses((const uint8_t*)arena_dev, off_dev, (const uint64_t*)(sd + o_len), n, kFusedMaxOutputs, (b200tfs_output*)(d + L.outs),
                            (int32_t*)(d + L.nouts), (b200tfs_model_spec*)(d + L.specs), (int32_t*)(d + L.status), nullptr, 0u,
                            (uint32_t*)(d + L.spill), c->stream));
  ConcatPlan cp{};
  cp.w = (const uint8_t*)arena_dev; cp.rec_off = off_dev; cp.outs = (const b200tfs_output*)(d + L.outs);
  cp.n_outs = (const int32_t*)(d + L.nouts); cp.rec_status = (const int32_t*)(d + L.status);
  cp.n = (uint32_t)n; cp.n_keys = (uint32_t)n_keys; cp.out_stride = kFusedMaxOutputs + 1; cp.cast = c->decode_cast;
  cp.kst = (int32_t*)(d + L.kst); cp.match = (int32_t*)(d + L.match);
  cp.vouts = (b200tfs_output*)(d + L.vouts); cp.vn_outs = (int32_t*)(d + L.vnouts); cp.vrec_status = (int32_t*)(d + L.vstatus);
  const VarPadMap* pad = nullptr;
  if ((rc = plan(cp, d, L, sd + o_keys, (const uint64_t*)(sd + o_len), &pad))) return rc;
  // packed-varint outputs: the single-launch decode's plan / count / emit over the table the plan kernel wrote (dst 0, stride 0)
  VarPlan vp{};
  vp.outs = cp.vouts; vp.n_outs = cp.vn_outs; vp.rec_status = cp.vrec_status;
  vp.w = cp.w; vp.rec_off = off_dev;
  vp.dst = nullptr; vp.dst_stride = 0; vp.n = (uint32_t)n; vp.tile_cap = (uint32_t)var_tile_cap;
  if ((rc = launch_varint_tail(c, vp, d + L.var, rec_off, pad))) return rc;
  if (slot->done && !c->capturing) { CU(cudaEventRecord(slot->done, c->stream)); slot->pending = true; }   // the kernels read the upload
  c->launches += 3;
  res.n = n; res.k = n_keys;
  res.vouts = L.vouts; res.vstat = L.var_status; res.specs = L.specs; res.status = L.status;
  return B200TFS_OK;
}

// b200tfs_decode_concat_host_async / b200tfs_decode_padded_host_async: the wire staged on the device, then `decode` (`name`)
template <class Key>
static int key_decode_host_async(b200tfs_ctx* c, const void* wire_host, int32_t n, const uint64_t* rec_off, const uint64_t* rec_len,
                                 int32_t n_keys, const Key* keys, const char* name,
                                 int (*decode)(b200tfs_ctx*, const void*, int32_t, const uint64_t*, const uint64_t*, int32_t, const Key*)) {
  if (!c || n <= 0 || !wire_host || !rec_off || !rec_len) return fail(B200TFS_E_ARG, "bad arguments");
  if (c->capturing) return fail(B200TFS_E_ARG, "capture %s over a device arena instead", name);
  CU(cudaSetDevice(c->device));
  uint64_t span;
  int rc = stage_wire(c, wire_host, n, rec_off, rec_len, &span);
  if (rc) return rc;
  return decode(c, c->stage_dev.p, n, rec_off, rec_len, n_keys, keys);
}
}  // extern "C++"

int b200tfs_decode_concat(b200tfs_ctx* c, const void* arena_dev, int32_t n, const uint64_t* rec_off, const uint64_t* rec_len,
                          int32_t n_keys, const b200tfs_concat_key* keys) {
  return b200tfs_decode_concat_strings(c, arena_dev, n, rec_off, rec_len, n_keys, keys, nullptr);
}

int b200tfs_decode_concat_strings(b200tfs_ctx* c, const void* arena_dev, int32_t n, const uint64_t* rec_off, const uint64_t* rec_len,
                                  int32_t n_keys, const b200tfs_concat_key* keys, const b200tfs_concat_strings* strings) {
  uint64_t var_tile_cap = 0, tile_cap = 0;
  int rc = key_begin(c, arena_dev, n, rec_off, rec_len, n_keys, keys, &var_tile_cap, [&](const b200tfs_concat_key&, int k) -> int {
    if (strings && strings[k].data_cap && !strings[k].data) return fail(B200TFS_E_ARG, "key %d: string data is NULL", k);
    return B200TFS_OK;
  });
  if (rc) return rc;
  const uint32_t vpt = decode_vpt(c, n, rec_len);
  for (int i = 0; i < n; ++i) tile_cap += concat_record_tile_bound(rec_len[i], 16ull * vpt, (uint32_t)n_keys);
  if (tile_cap > 0x7FFFFFFFull) return fail(B200TFS_E_TOOBIG, "batch needs more than 2^31 tiles");
  const PlanGeometry g = plan_geometry((uint64_t)n * (uint64_t)n_keys * B200TFS_MAX_RUNS, tile_cap, 0);   // concat_plan_kernel's plan image
  if (g.off_tiles > 0xFFFFFFFFull) return fail(B200TFS_E_TOOBIG, "plan image larger than 4 GiB");
  // the string pairs' scratch: bytes | data0 | chunk0 (n_keys * n each) | n_chunks
  const uint64_t pairs = (uint64_t)n * (uint64_t)n_keys, str_bytes = 24 * pairs + 8;
  uint64_t chunk_bound = 0;
  for (int i = 0; strings && i < n; ++i) chunk_bound += (uint64_t)n_keys * (str_count_bound(rec_len[i]) / kStrChunk + 1);
  const auto plan = [&](ConcatPlan& cp, uint8_t* d, const KeyLayout& L, const uint8_t* kd, const uint64_t* len_dev, const VarPadMap**) -> int {
    cp.keys = (const ConcatKeyDev*)kd; cp.vpt = vpt; cp.tile_cap = (uint32_t)tile_cap; cp.plan = d + L.own[0];
    CU(launch_concat_plan(cp, (uint32_t)tile_cap, c->stream, strings != nullptr));
    if (!strings) return B200TFS_OK;
    StrTables T{};
    for (int k = 0; k < n_keys; ++k) T.keys[k] = StrKeyDev{(uint8_t*)strings[k].data, strings[k].data_cap};
    T.w = cp.w; T.rec_off = cp.rec_off; T.rec_len = len_dev; T.vouts = cp.vouts;
    T.bytes = (uint64_t*)(d + L.own[1]); T.data0 = T.bytes + pairs; T.chunk0 = T.data0 + pairs; T.n_chunks = T.chunk0 + pairs;
    T.n = (uint32_t)n; T.n_keys = (uint32_t)n_keys;
    const uint64_t grid = std::min<uint64_t>((chunk_bound + kStrThreads / 32 - 1) / (kStrThreads / 32), (uint64_t)c->sm_count * 8);
    CU(launch_concat_strings(T, (uint32_t)grid, c->stream));
    c->launches += 4;
    return B200TFS_OK;
  };
  const auto dev_key = [](const b200tfs_concat_key& k, const uint8_t* kb) { return ConcatKeyDev{kb, (uint8_t*)k.dst, k.dst_cap, (uint32_t)k.key_len, 0u}; };
  if (strings)
    return key_decode(c, c->concat_dev, c->concat_res, arena_dev, n, rec_off, rec_len, n_keys, keys, var_tile_cap, {g.end, str_bytes}, dev_key, plan);
  return key_decode(c, c->concat_dev, c->concat_res, arena_dev, n, rec_off, rec_len, n_keys, keys, var_tile_cap, {g.end}, dev_key, plan);
}

int b200tfs_decode_concat_host_async(b200tfs_ctx* c, const void* wire_host, int32_t n, const uint64_t* rec_off, const uint64_t* rec_len,
                                     int32_t n_keys, const b200tfs_concat_key* keys) {
  return key_decode_host_async(c, wire_host, n, rec_off, rec_len, n_keys, keys, "b200tfs_decode_concat", b200tfs_decode_concat);
}

int b200tfs_decode_concat_strings_host_async(b200tfs_ctx* c, const void* wire_host, int32_t n, const uint64_t* rec_off,
                                             const uint64_t* rec_len, int32_t n_keys, const b200tfs_concat_key* keys,
                                             const b200tfs_concat_strings* strings) {
  if (!c || n <= 0 || !wire_host || !rec_off || !rec_len) return fail(B200TFS_E_ARG, "bad arguments");
  if (c->capturing) return fail(B200TFS_E_ARG, "capture b200tfs_decode_concat_strings over a device arena instead");
  CU(cudaSetDevice(c->device));
  uint64_t span;
  int rc = stage_wire(c, wire_host, n, rec_off, rec_len, &span);
  if (rc) return rc;
  return b200tfs_decode_concat_strings(c, c->stage_dev.p, n, rec_off, rec_len, n_keys, keys, strings);
}

// The results of a per-key decode (`R` of its most recent call, its scratch at `base`), as b200tfs_concat_results describes them
static int key_results(b200tfs_ctx* c, const b200tfs_ctx::KeyResults& R, const uint8_t* base, const char* what, int32_t n, int32_t n_keys,
                       b200tfs_output* outs, b200tfs_model_spec* specs, int32_t* rec_status) {
  if (!c || n < 0 || n_keys < 0) return fail(B200TFS_E_ARG, "bad arguments");
  if (c->capturing) return fail(B200TFS_E_ARG, "cannot collect results during graph capture");
  if (n != R.n || n_keys != R.k) return fail(B200TFS_E_ARG, "the last %s had %d records and %d keys", what, R.n, R.k);
  if (n == 0) return B200TFS_OK;
  CU(cudaSetDevice(c->device));
  CU(cudaStreamSynchronize(c->stream));
  const uint8_t* d = base;
  if (outs) {
    std::vector<b200tfs_output> v((size_t)n * kFusedMaxOutputs);
    std::vector<int32_t> vs((size_t)n * kFusedMaxOutputs);
    CU(cudaMemcpy(v.data(), d + R.vouts, sizeof(b200tfs_output) * v.size(), cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(vs.data(), d + R.vstat, 4 * vs.size(), cudaMemcpyDeviceToHost));
    for (int r = 0; r < n; ++r)
      for (int k = 0; k < n_keys; ++k) {
        b200tfs_output o = v[(size_t)r * kFusedMaxOutputs + k];
        fold_varint_status(o, vs[(size_t)r * kFusedMaxOutputs + k]);
        o.dst_off -= (uint64_t)(uintptr_t)R.dst[k];
        outs[(size_t)r * n_keys + k] = o;
      }
  }
  if (specs) CU(cudaMemcpy(specs, d + R.specs, sizeof(b200tfs_model_spec) * (uint64_t)n, cudaMemcpyDeviceToHost));
  if (rec_status) {
    CU(cudaMemcpy(rec_status, d + R.status, 4ull * n, cudaMemcpyDeviceToHost));
    for (int r = 0; r < n; ++r) if (rec_status[r] == B200TFS_E_SPILL || rec_status[r] == B200TFS_E_SIZE) rec_status[r] = B200TFS_E_NONCANONICAL;
  }
  return B200TFS_OK;
}

int b200tfs_concat_results(b200tfs_ctx* c, int32_t n, int32_t n_keys, b200tfs_output* outs, b200tfs_model_spec* specs, int32_t* rec_status) {
  if (!c) return fail(B200TFS_E_ARG, "bad arguments");
  return key_results(c, c->concat_res, (const uint8_t*)c->concat_dev.p, "b200tfs_decode_concat", n, n_keys, outs, specs, rec_status);
}

// ------------------------------------------------------------------------------------------------
// decode into one padded tensor per key
// ------------------------------------------------------------------------------------------------
int b200tfs_decode_padded(b200tfs_ctx* c, const void* arena_dev, int32_t n, const uint64_t* rec_off, const uint64_t* rec_len,
                          int32_t n_keys, const b200tfs_pad_key* keys) {
  return b200tfs_decode_padded_strings(c, arena_dev, n, rec_off, rec_len, n_keys, keys, nullptr);
}

int b200tfs_decode_padded_strings(b200tfs_ctx* c, const void* arena_dev, int32_t n, const uint64_t* rec_off, const uint64_t* rec_len,
                                  int32_t n_keys, const b200tfs_pad_key* keys, const b200tfs_padded_strings* strings) {
  uint64_t var_tile_cap = 0, chunk_bound = 0, pos_bound = 0;
  int rc = key_begin(c, arena_dev, n, rec_off, rec_len, n_keys, keys, &var_tile_cap, [&](const b200tfs_pad_key& K, int k) -> int {
    if (strings && strings[k].data_cap && !strings[k].data) return fail(B200TFS_E_ARG, "key %d: string data is NULL", k);
    if (strings && strings[k].pad_len && !strings[k].pad) return fail(B200TFS_E_ARG, "key %d: pad string is NULL", k);
    pos_bound += K.dst_cap / 8;
    if ((uintptr_t)K.dst & 15) return fail(B200TFS_E_ARG, "key %d: dst is not 16-byte aligned", k);
    if (K.rank < 1 || K.rank > B200TFS_MAX_RANK) return fail(B200TFS_E_ARG, "key %d: rank %d", k, K.rank);
    uint64_t row = 1;
    for (int d = 1; d < K.rank; ++d) {
      if (K.dims[d] < 0 || (K.dims[d] && row > 0xFFFFFFFFull / (uint64_t)K.dims[d])) return fail(B200TFS_E_ARG, "key %d: a row holds 2^32 elements or more", k);
      row *= (uint64_t)K.dims[d];
    }
    chunk_bound += (K.dst_cap + kPadChunkBytes - 1) / kPadChunkBytes;
    return B200TFS_OK;
  });
  if (rc) return rc;
  const uint64_t pairs = (uint64_t)n * (uint64_t)n_keys;
  VarPadMap pm{};
  HostBytes pads[B200TFS_CONCAT_MAX_KEYS];   // the pad strings, uploaded with the keys
  for (int k = 0; strings && k < n_keys; ++k) pads[k] = HostBytes{strings[k].pad, strings[k].pad_len, nullptr};
  const auto plan = [&](ConcatPlan& cp, uint8_t* d, const KeyLayout& L, const uint8_t* kd, const uint64_t* len_dev, const VarPadMap** pad) -> int {
    PaddedPlan pp{};
    pp.cp = cp;
    pp.keys = (const PadKeyDev*)kd;
    pp.desc = (PadDesc*)(d + L.own[0]); pp.first_row = (uint64_t*)(d + L.own[1]); pp.kout = (PadKeyOut*)(d + L.own[2]);
    const uint32_t emit_grid = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>(chunk_bound, (uint64_t)c->sm_count * 8));
    CU(launch_padded(pp, emit_grid, c->stream, strings != nullptr));
    // the varint emit stores every element at its padded position
    pm = VarPadMap{pp.desc, pp.keys, (uint32_t)n_keys, 0u};
    *pad = &pm;
    if (!strings) return B200TFS_OK;
    PadStrTables T{};
    T.pp = pp;
    T.rec_len = len_dev;
    for (int k = 0; k < n_keys; ++k) T.keys[k] = PadStrKeyDev{(uint8_t*)strings[k].data, strings[k].data_cap, pads[k].dev, pads[k].len};
    T.bytes = (uint64_t*)(d + L.own[3]); T.data0 = T.bytes + pairs; T.pos0 = T.data0 + pairs;
    const uint64_t grid = std::min<uint64_t>((pos_bound + kStrThreads - 1) / kStrThreads, (uint64_t)c->sm_count * 8);
    CU(launch_padded_strings(T, (uint32_t)grid, c->stream));
    c->launches += 4;
    return B200TFS_OK;
  };
  const auto dev_key = [](const b200tfs_pad_key& k, const uint8_t* kb) {
    PadKeyDev kd{};
    kd.k = ConcatKeyDev{kb, (uint8_t*)k.dst, k.dst_cap, (uint32_t)k.key_len, 0u};
    for (int d = 0; d < B200TFS_MAX_RANK; ++d) kd.dims[d] = k.dims[d];
    memcpy(kd.pad, k.pad_bits, 16);
    kd.rank = k.rank;
    return kd;
  };
  if (strings)   // the string pairs' scratch: bytes | data0 (n_keys * n each) | pos0 (n_keys + 1)
    return key_decode(c, c->padded_dev, c->padded_res, arena_dev, n, rec_off, rec_len, n_keys, keys, var_tile_cap,
                      {sizeof(PadDesc) * pairs, 8 * pairs, sizeof(PadKeyOut) * (n_keys + 1), 16 * pairs + 8ull * (n_keys + 1)}, dev_key, plan,
                      pads, n_keys);
  return key_decode(c, c->padded_dev, c->padded_res, arena_dev, n, rec_off, rec_len, n_keys, keys, var_tile_cap,
                    {sizeof(PadDesc) * pairs, 8 * pairs, sizeof(PadKeyOut) * (n_keys + 1)}, dev_key, plan);
}

int b200tfs_decode_padded_host_async(b200tfs_ctx* c, const void* wire_host, int32_t n, const uint64_t* rec_off, const uint64_t* rec_len,
                                     int32_t n_keys, const b200tfs_pad_key* keys) {
  return key_decode_host_async(c, wire_host, n, rec_off, rec_len, n_keys, keys, "b200tfs_decode_padded", b200tfs_decode_padded);
}

int b200tfs_decode_padded_strings_host_async(b200tfs_ctx* c, const void* wire_host, int32_t n, const uint64_t* rec_off,
                                             const uint64_t* rec_len, int32_t n_keys, const b200tfs_pad_key* keys,
                                             const b200tfs_padded_strings* strings) {
  if (!c || n <= 0 || !wire_host || !rec_off || !rec_len) return fail(B200TFS_E_ARG, "bad arguments");
  if (c->capturing) return fail(B200TFS_E_ARG, "capture b200tfs_decode_padded_strings over a device arena instead");
  CU(cudaSetDevice(c->device));
  uint64_t span;
  int rc = stage_wire(c, wire_host, n, rec_off, rec_len, &span);
  if (rc) return rc;
  return b200tfs_decode_padded_strings(c, c->stage_dev.p, n, rec_off, rec_len, n_keys, keys, strings);
}

int b200tfs_padded_results(b200tfs_ctx* c, int32_t n, int32_t n_keys, b200tfs_output* outs, b200tfs_model_spec* specs, int32_t* rec_status) {
  if (!c) return fail(B200TFS_E_ARG, "bad arguments");
  return key_results(c, c->padded_res, (const uint8_t*)c->padded_dev.p, "b200tfs_decode_padded", n, n_keys, outs, specs, rec_status);
}

}  // extern "C"

// The checks a string column's b200tfs_bytes entry takes in every route that reads one (B200TFS_E_ARG).  `what` and the arguments
// behind it, a printf format such as "input %d", name the column in the message; they are formatted only for a refusal.
static int bytes_entry_check(const b200tfs_bytes& b, const void* data, const char* what, ...) {
  char msg[64];
  if (b.flags & ~B200TFS_F_DEVICE_DATA) snprintf(msg, sizeof msg, "unknown bytes flags 0x%x", (unsigned)b.flags);
  else if (b.data_len < 0) snprintf(msg, sizeof msg, "negative data_len %lld", (long long)b.data_len);
  else if (b.data_len && !data) snprintf(msg, sizeof msg, "data pointer is NULL");
  else if ((uintptr_t)b.offsets & 7) snprintf(msg, sizeof msg, "string offsets must be 8-byte aligned");
  else return B200TFS_OK;
  char name[64];
  va_list ap;
  va_start(ap, what);
  vsnprintf(name, sizeof name, what, ap);
  va_end(ap);
  return fail(B200TFS_E_ARG, "%s: %s", name, msg);
}

// ------------------------------------------------------------------------------------------------
// varint dtypes (phase 2: kernels in kernels.cu; wired here)
// ------------------------------------------------------------------------------------------------
#include "varint_host.inc"
#include "example_host.inc"
#include "unpad_host.inc"
