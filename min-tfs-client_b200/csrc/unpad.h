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
  uint32_t str;                    // string input str - 1 (0: none) - a DT_STRING column (b200tfs_bytes), its offsets and data_len in
                                   // UnpadPlan::str_cols: src is its byte buffer, element e is string e (src_esz 1, so a box's
                                   // src_off counts strings), field F_STRING
};

struct UnpadStrCol {               // the offsets of a string input (kept out of UnpadIn, which the varint kernels copy per thread)
  const int64_t* offsets;          // device int64[strings + 1]
  int64_t data_len;                // bytes of the input's src
};

struct UnpadBox {                  // one (request, input)
  int64_t dims[B200TFS_MAX_RANK];  // the request's shape for the input
  uint64_t src_off;                // byte offset of its first element in the source (string column: index of its first string)
  uint64_t n_elems;
  uint64_t run, n_runs;            // n_runs runs of `run` elements (see above); n_runs <= 1: one contiguous stretch
  uint64_t payload;                // wire bytes of its values (varints: the counted total; strings: sum of 1 + vi(len) + len)
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

// ---- string columns --------------------------------------------------------------------------------------------------------
// A box of a string column reads, in element order, the offset of its first row's start, both ends of every string of the box and
// its last row's end; these must never decrease and stay within [0, data_len] (a broadcast input reads every offset).  When every
// request of the call follows the rule, the boxes take disjoint byte ranges and the padded inputs' strings fit in data_len bytes.
// The count and emit kernels see every offset through unpad_str_off: clamped into [0, data_len], so both agree on every length
// whatever the offsets hold and no read leaves the buffer; a box whose offsets break the rule gets B200TFS_E_SHAPE and writes
// nothing.  Such a request can also let the good ones on either side of it read overlapping bytes (its last row's end below its
// first row's start), so that together they need more than the arena bound: the layout kernel's arena_cap check then gives the
// later ones B200TFS_E_SIZE instead of their bytes - never a store outside the good records.
B2_HD uint64_t unpad_str_off(const UnpadStrCol& c, uint64_t i, bool* ok) {
  const int64_t v = c.offsets[i];
  if (v < 0 || v > c.data_len) *ok = false;
  return v < 0 ? 0 : v > c.data_len ? (uint64_t)c.data_len : (uint64_t)v;
}
// column index of string e of box b (src_off: the box's first string)
B2_HD uint64_t unpad_str_index(const UnpadIn& in, const UnpadBox& b, uint64_t e) {
  if (b.n_runs <= 1) return b.src_off + e;
  const uint64_t q = e / b.run;
  return b.src_off + unpad_run_start(in, b, q) + (e - q * b.run);
}
// the offset indexes of box b's first row's start and last row's end (broadcast: the whole column)
B2_HD void unpad_str_rows(const UnpadIn& in, const UnpadBox& b, uint64_t* first, uint64_t* end) {
  uint64_t w = 1;
  for (int32_t d = 1; d < in.rank; ++d) w *= (uint64_t)in.dims[d];
  *first = in.shapes ? b.src_off : 0;
  *end = in.shapes ? b.src_off + (uint64_t)b.dims[0] * w : b.n_elems;
}

struct UnpadFrame {                // what every request's framing has in common
  const uint8_t* blob;             // model_spec field (its tag included) at 0, the output_filter run, then the keys
  uint32_t spec_len, grpc;         // grpc: gRPC's 5-byte length-prefixed-message header in front
  uint32_t n_in, tail_len;         // tail_len: bytes of the output_filter run
};

// write_request's view of one request of the padded encode: every input from its box, payloads skipped
struct UnpadRequest {
  const UnpadFrame& F;
  const UnpadIn* ins;
  const UnpadBox* box;
  uint64_t* payload_off;           // may be null
  uint64_t o0;
  template <class Out> B2_HD void spec(Out& o) { o.bytes(F.blob, F.spec_len); }
  template <class Out> B2_HD void tail(Out& o) { o.bytes(F.blob + F.spec_len, F.tail_len); }
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
  // string jobs (request r, string input k: r * n_str + k), in tables of their own shaped like the varint ones: a tile is
  // kVarThreads strings, tile_val its wire bytes (saturated at 2^32 - 1), total the box's payload
  uint32_t n_str, str_tile_cap, str_group_cap, pad2_;
  uint8_t str_in[kUnpadMaxInputs]; // input index of string input k
  const UnpadStrCol* str_cols;     // [n_str]
  VarJobDev* str_jobs;             // [n * n_str]
  uint32_t* str_tile_job;          // [str_tile_cap]
  uint32_t* str_tile_val;          // [str_tile_cap]
  uint32_t* str_group_sum;         // [str_group_cap]
  unsigned long long* str_total;   // [n * n_str]
  uint32_t* n_str_tiles;           // [1]
  // move plan: PlanHeader | MoveItem[item_cap] | TileRef[tile_cap]
  uint8_t* plan;
  uint32_t item_cap, tile_cap, vpt, pad_;
  uint64_t* rec_off_host; uint64_t* rec_len_host; int32_t* status_host;   // pinned: read by b200tfs_encode_results
};

}  // namespace b200tfs
