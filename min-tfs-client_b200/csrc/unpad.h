// unpad.h - b200tfs_encode_padded_requests_async: n PredictRequests cut out of one padded tensor per input.  What the plan kernel,
// the framing kernels (unpad_kernels.cuh) and the host emulation (b200tfs_padded_request_frame) share: the per-input table the
// host fixes, the box of one (request, input) and the framing of one request, written through framing.h.
//
// Request r's tensor for input j is the box P_j[r0 : r0 + S[r,0], :S[r,1], ..., :S[r,m-1]] with r0 the rows of requests 0..r-1.
// A box is `n_runs` runs of `run` consecutive source elements: its axes from `lo` on are one contiguous stretch of the padded
// tensor (every axis after `lo` is full), the axes before `lo` index the runs.
#pragma once
#include <stdint.h>

#include "../../include/b200tfs.h"
#include "framing.h"
#include "plan.h"
#include "wire.h"

namespace b200tfs {

constexpr uint32_t kUnpadMaxInputs = 2 * B200TFS_CONCAT_MAX_KEYS;   // padded inputs + broadcast inputs of one call
constexpr uint32_t kUnpadFrameThreads = 128;                        // requests per framing CTA (one thread each)

struct UnpadIn {                   // one input of every request, in wire (key) order
  const uint8_t* src;              // the padded tensor (broadcast: the tensor), device
  const int64_t* shapes;           // device int64[n, cols]; nullptr for a broadcast input
  int64_t dims[B200TFS_MAX_RANK];  // the padded tensor's dims (broadcast: the tensor's own)
  int32_t rank, cols;              // cols: rank (full shapes) or 1 (row counts)
  int32_t wire_dtype;
  uint32_t flags;                  // B200TFS_F_* of the tensor header (only F_PRESERIALIZED matters to it: never set here)
  uint32_t op;                     // MoveOp of a fixed-width payload
  uint32_t src_esz, wire_esz;      // element size in memory / wire bytes per element (fixed width and bool)
  uint32_t varint, is_signed, field;
  uint32_t key_off, key_len;       // key bytes in the blob
  uint32_t pad_;
};

struct UnpadBox {                  // one (request, input)
  int64_t dims[B200TFS_MAX_RANK];  // the request's shape for the input
  uint64_t src_off;                // byte offset of its first element in the source
  uint64_t n_elems;
  uint64_t run, n_runs;            // n_runs runs of `run` elements (see above); n_runs <= 1: one contiguous stretch
  uint64_t payload;                // wire bytes of its values (varints: the counted total)
  uint32_t lo, pad_;
};

// the request's shape for `in` from its row of the shapes table (broadcast: the input's dims), checked against the padded tensor:
// B200TFS_OK or B200TFS_E_SHAPE (a negative dim, a trailing dim past the padded one).  src_off is the caller's (it needs the rows in
// front); the element count and the run geometry are filled in here.
B2_HD int32_t unpad_box(const UnpadIn& in, const int64_t* row, UnpadBox* b) {
  int32_t st = B200TFS_OK;
  for (int32_t d = 0; d < in.rank; ++d) {
    int64_t x = in.dims[d];
    if (in.shapes && (d == 0 || in.cols > 1)) x = row[d];
    if (x < 0 || (in.shapes && d > 0 && x > in.dims[d])) { st = B200TFS_E_SHAPE; x = 0; }
    b->dims[d] = x;
  }
  uint64_t n = 1;
  for (int32_t d = 0; d < in.rank; ++d) n *= (uint64_t)b->dims[d];
  b->n_elems = st == B200TFS_OK ? n : 0;
  int32_t lo = in.rank;                          // the contiguous tail: axes lo.. with every axis after lo full
  uint64_t run = 1;
  while (lo > 0) {
    --lo;
    run *= (uint64_t)b->dims[lo];
    if (b->dims[lo] != in.dims[lo]) break;
  }
  b->lo = (uint32_t)lo;
  b->run = run;
  b->n_runs = run ? b->n_elems / run : 0;
  b->payload = 0;
  return st;
}

// source element offset (in elements, from the box's first one) of the first element of run q
B2_HD uint64_t unpad_run_start(const UnpadIn& in, const UnpadBox& b, uint64_t q) {
  uint64_t off = 0, pitch = 1;
  for (int32_t d = in.rank - 1; d >= (int32_t)b.lo; --d) pitch *= (uint64_t)in.dims[d];   // elements of one index of axis lo - 1
  for (int32_t d = (int32_t)b.lo - 1; d >= 0; --d) {
    const uint64_t x = (uint64_t)b.dims[d], i = q % x;
    q /= x;
    off += i * pitch;
    pitch *= (uint64_t)in.dims[d];
  }
  return off;
}

struct UnpadFrame {                // what every request's framing has in common
  const uint8_t* blob;             // model_spec field (its tag included) at 0, then the keys
  uint32_t spec_len, grpc;         // grpc: gRPC's 5-byte length-prefixed-message header in front
  uint32_t n_in, pad_;
};

// write_request's view of one request of the padded encode: every input from its box, payloads skipped
struct UnpadRequest {
  const UnpadFrame& F;
  const UnpadIn* ins;
  const UnpadBox* box;
  uint64_t* payload_off;           // may be null
  uint64_t o0;
  template <class Out> B2_HD void spec(Out& o) { o.bytes(F.blob, F.spec_len); }
  B2_HD void input(uint32_t j, b200tfs_tensor& t, TensorLayout& L) const {
    const UnpadIn& in = ins[j];
    t.wire_dtype = in.wire_dtype; t.rank = in.rank; t.flags = in.flags; t.dims = box[j].dims;
    t.key = (const char*)F.blob + in.key_off; t.key_len = in.key_len;
    L.payload_len = box[j].payload; L.field = in.field; L.shape_len = shape_body_len(in.rank, box[j].dims);
  }
  template <class Out> B2_HD void payload(Out& o, uint32_t j, const b200tfs_tensor&, const TensorLayout& L) {
    if (payload_off) payload_off[j] = o.pos() - o0;
    o.skip(L.payload_len);
  }
};

// The framing of one request through `o`, payloads skipped.  The box payloads must be set; `msg` is the message length
// (unpad_layout).  payload_off (may be null) receives where each input's payload starts, counted from the first byte written.
template <class Out>
B2_HD void unpad_write(Out& o, const UnpadFrame& F, const UnpadIn* ins, const UnpadBox* box, uint64_t msg, uint64_t* payload_off) {
  UnpadRequest q{F, ins, box, payload_off, o.pos()};
  write_request(o, q, F.n_in, F.grpc != 0, msg);
}

// Length of the record (gRPC prefix included) and, per input, where its payload starts; *largest_off: the start of the largest
// payload (placement aligns it to 128 bytes).  0 with *st = B200TFS_E_TOOBIG for a message or TensorProto over 2 GiB.
B2_HD uint64_t unpad_layout(const UnpadFrame& F, const UnpadIn* ins, const UnpadBox* box, uint64_t* payload_off, uint64_t* largest_off,
                            int32_t* st) {
  CountOut c;
  unpad_write(c, F, ins, box, 0, payload_off);     // the prefix's length does not depend on its value
  const uint64_t msg = c.n - (F.grpc ? 5 : 0);
  uint64_t largest = 0;
  *largest_off = 0;
  bool big = msg > 0x7FFFFFFFull;
  for (uint32_t j = 0; j < F.n_in; ++j) {
    if (box[j].payload > largest) { largest = box[j].payload; *largest_off = payload_off[j]; }
    if (box[j].payload > 0x7FFFFFFFull) big = true;
  }
  *st = big ? B200TFS_E_TOOBIG : B200TFS_OK;
  return big ? 0 : c.n;
}

// ---- the device launch (unpad_kernels.cuh) -----------------------------------------------------------------------------------
struct UnpadPlan {
  const UnpadIn* ins;              // [n_in], wire order
  UnpadFrame F;
  uint32_t n, n_var;               // requests; packed-varint inputs (job of request r, varint input v: r * n_var + v)
  uint8_t var_in[kUnpadMaxInputs]; // input index of varint input v
  uint8_t* arena;
  uint64_t arena_cap;
  UnpadBox* box;                   // [n * n_in]
  int32_t* st;                     // [n] request status
  uint64_t* rec_off;               // [n] device copies of the results, for the framing kernel
  // packed-varint jobs
  VarJobDev* jobs;                 // [n * n_var]
  uint32_t* tile_job;              // [var_tile_cap]
  uint32_t* tile_val;              // [var_tile_cap]
  uint32_t* group_sum;             // [var_group_cap]: every job's ceil(tiles / kVarGroupTiles) groups, scanned apart
  unsigned long long* total;       // [n * n_var]
  uint32_t* n_var_tiles;           // [1]
  uint32_t var_tile_cap, var_group_cap;
  // move plan: PlanHeader | MoveItem[item_cap] | TileRef[tile_cap]
  uint8_t* plan;
  uint32_t item_cap, tile_cap, vpt, pad_;
  uint64_t* rec_off_host; uint64_t* rec_len_host; int32_t* status_host;   // pinned: read by b200tfs_encode_results
};

}  // namespace b200tfs
