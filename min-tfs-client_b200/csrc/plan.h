// plan.h - the launch plan shared by the host planner (codec_host.cpp) and the kernels (kernels.cu).
//
// A plan is a flat byte image: PlanHeader, then MoveItem[n_items], TileRef[n_tiles] (absent when
// uniform_tpi != 0), SmallItem[n_small], then the header blob (the varint tags / lengths / dims /
// keys the planner computed - the non-payload bytes of the wire).  It reaches the kernel either
// by value in the kernel parameter space (<= kInlinePlanBytes, no copy at all: the C2 single-tensor
// case) or through one pinned-host -> device copy.
#pragma once
#include <stdint.h>

#include "../../include/b200tfs.h"
#include "wire.h"

namespace b200tfs {

// what a MoveItem / SmallItem does to the bytes it moves
enum MoveOp : uint32_t {
  OP_COPY = 0,        // raw little-endian bytes (float64, complex, tensor_content, KEEP_SNAN float32)
  OP_QUIET_SRC = 1,   // float32 sNaN -> qNaN, 4-byte elements aligned with the SOURCE start (encode)
  OP_QUIET_DST = 2,   // same, elements aligned with the DESTINATION start (decode)
  OP_BOOL = 3,        // byte != 0 -> 1 (bool_val written from numpy bool memory)
  OP_H2F = 4,         // float16  -> float32 (exact), encode-side cast
  OP_B2F = 5,         // bfloat16 -> float32 (exact), encode-side cast
  OP_F2H = 6,         // float32 -> float16, round-to-nearest-even, decode-side cast
  OP_F2B = 7,         // float32 -> bfloat16, round-to-nearest-even, decode-side cast
  OP_FLAG_BLOB = 0x80000000u  // SmallItem: src is an offset into the plan image, not a pointer
};

struct MoveItem {     // one large payload, tiled across CTAs
  const uint8_t* src;
  uint8_t* dst;
  uint64_t n_out;     // bytes written
  uint32_t op;
  uint32_t n_tiles;   // max(1, ceil(ceil(n_out/16) / vec_per_tile))
  uint32_t glen, gstride;  // gstride != 0: the source is a row of pieces, `glen` value bytes every `gstride` bytes (a run of
                           // unpacked elements, b200tfs_run): logical source byte j lies at src[(j / glen) * gstride + j % glen]
};

struct TileRef { uint32_t item; uint32_t tile; };

struct SmallItem {    // one header fragment or small payload: a warp moves it
  uint64_t src;       // pointer, or offset into the plan image with OP_FLAG_BLOB
  uint8_t* dst;
  uint32_t n_out;
  uint32_t op;
  uint32_t glen, gstride;  // as in MoveItem
};

struct PlanHeader {
  uint32_t n_items, n_tiles, n_small, uniform_tpi;  // uniform_tpi: every item has this many tiles (no TileRef table)
  uint32_t vec_per_tile;                            // 16-byte vectors of destination per tile
  uint32_t off_items, off_tiles, off_small;         // byte offsets inside the plan image
  uint32_t guard_div;                               // move_guarded_kernel: item i is stored only if guard[i / guard_div] != 0
  uint32_t independent;                             // != 0: nothing in this plan is written by the kernel launched just before (the framing
                                                    // kernel of a deferred encode whose movers all have host-fixed destinations): no wait for it
  uint32_t pad[2];
  const uint32_t* guard;
};

#if defined(__CUDACC__)
#define B2_PLAN_HD __host__ __device__ __forceinline__
#else
#define B2_PLAN_HD inline
#endif

// Where the tables of a plan image lie: PlanHeader | MoveItem[n_items] | TileRef[n_tile_refs] | SmallItem[n_small], and `end`,
// where the header blob starts.  The host planner (build_plan), the scratch sizing of b200tfs_decode_concat and
// concat_plan_kernel, which writes such an image on the device, all take it from here.
struct PlanGeometry { uint64_t off_items, off_tiles, off_small, end; };
B2_PLAN_HD PlanGeometry plan_geometry(uint64_t n_items, uint64_t n_tile_refs, uint64_t n_small) {
  PlanGeometry g;
  g.off_items = (sizeof(PlanHeader) + 15) & ~15ull;
  g.off_tiles = g.off_items + n_items * sizeof(MoveItem);
  g.off_small = (g.off_tiles + n_tile_refs * sizeof(TileRef) + 15) & ~15ull;
  g.end = g.off_small + n_small * sizeof(SmallItem);
  return g;
}

constexpr uint32_t kInlinePlanBytes = 3840;  // fits the classic 4 KB kernel-parameter window
struct InlinePlan { uint8_t bytes[kInlinePlanBytes]; };

constexpr uint32_t kMoveThreads = 256;      // threads per CTA of move_kernel
constexpr uint32_t kSmallMax = 2048;        // payloads up to this many bytes take the warp path

// ---- fused single-launch decode ---------------------------------------------------------------
constexpr int kFusedMaxOutputs = 8;    // outputs tabulated per record by decode_fused_kernel
constexpr int kFusedInlineRecs = 16;   // up to this many records travel in the kernel parameters
constexpr uint32_t kFusedSlackTiles = 8;  // tiles budgeted per record beyond ceil(rec_len / tile)

struct FusedInline { uint64_t off[kFusedInlineRecs], len[kFusedInlineRecs]; uint32_t tile_start[kFusedInlineRecs + 1]; };

// framing template left by one decode launch for the next (see decode_fused_kernel)
constexpr uint32_t kTplChunks = 4;
constexpr uint32_t kTplFraming = 256;   // == kMoveThreads: one framing byte per thread
struct TplChunk { uint32_t wire_off, len, dst_off, op, n_tiles, is_varint, fpos, pad; };  // record-relative
struct TplHead {
  uint32_t valid, n_chunks, n_outs, framing_len;
  uint64_t rec_len, dst_need;
  uint32_t vpt, total_tiles;
  uint32_t serial, cast;       // serial: which learning produced it (the table entries below belong to exactly this serial);
                               // cast: the float narrowing it was laid out for (0 / DT_HALF / DT_BFLOAT16: FusedParams::cast)
  uint32_t varints, pad;       // varints: laid out with ranges for the packed-varint outputs (FusedParams::varints)
};
// the part of a template every CTA needs before it can start on its tile: small enough to ride in the kernel parameters
// (no load at all ahead of the tile's loads) when the host knows it - because it walked record 0 itself (host-buffer entry
// points) or because an earlier launch left it in pinned memory and the stream has been idle since
struct TplInline {
  TplHead head;
  TplChunk chunk[kTplChunks];
  uint8_t framing[kTplFraming];
};
struct Template {
  TplInline in;
  b200tfs_model_spec spec;
  b200tfs_output outs[kFusedMaxOutputs];
};

struct FusedParams {
  const uint8_t* w;          // wire arena
  uint8_t* dst;              // destination base; record r owns [r*dst_stride, (r+1)*dst_stride)
  uint64_t dst_stride;
  int32_t n;
  uint32_t vpt;
  b200tfs_output* outs;      // device table, n * kFusedMaxOutputs
  int32_t* n_outs;
  b200tfs_model_spec* specs;
  int32_t* status;
  const uint32_t* cta_rec;   // n > kFusedInlineRecs: record of every CTA, tile_start[n+1], rec_off, rec_len
  const uint32_t* tile_start;
  const uint64_t* rec_off;
  const uint64_t* rec_len;
  const Template* tpl_read;  // template written by the previous launch on this context (may be invalid)
  Template* tpl_write;       // where record 0 of this launch leaves its template
  TplInline* tpl_pinned;     // pinned host copy of the inline part, written whenever a template is learnt (valid flag last)
  unsigned long long* stats; // device counters: records served by [0] the template in the parameters, [1] the device template, [2] the walk
  uint32_t serial;           // stamp for a template learnt by THIS launch
  uint32_t cast;             // DT_FLOAT outputs are narrowed on the way out: 0 = no, DT_HALF (19) / DT_BFLOAT16 (14) (b200tfs_set_decode_cast)
  uint32_t mode;             // 0: the whole decode.  The narrowing decode of a batch whose template the host knows runs as three launches:
                             // 1 = verify only (two CTAs per record: framing verdict -> guard[r], table), then move_guarded_kernel over a
                             // host-built plan, then 2 = the whole decode for the records whose guard is still 0 (the others leave at once)
  uint32_t* guard;
  uint32_t tile_bias;        // a SLICE of a one-record launch (the pipelined host path): CTA b works as CTA b + tile_bias of the full grid
  uint32_t trusted;          // != 0: the host built the inline template from THIS record's own bytes: no verdict (a slice's launch runs
                             // before the record's tail - and with it part of the framing - has arrived on the device)
  uint32_t varints;          // != 0: packed-varint outputs get ranges of the slot too (b200tfs_set_decode_varints; vdec_plan_kernel fills them)
  uint32_t pad;
  FusedInline inl;
  TplInline tpli;            // head.valid != 0: the template as the host knows it (tier 1; tpl_read is tier 2, the walk tier 3)
};

// ---- packed-varint jobs ------------------------------------------------------------------------
constexpr uint32_t kVarThreads = 256;
constexpr uint32_t kVarPerThread = 8;
constexpr uint32_t kVarTileElems = kVarThreads * kVarPerThread;  // elements per encode tile
constexpr uint32_t kVarTileBytes = kVarThreads * 32;             // wire bytes per decode tile; tiles are cut at 16-byte-aligned ADDRESSES
constexpr int32_t kVarFlagHalfAsValue = 1;  // decode half_val ints as VALUES (the reference's DT_HALF quirk, SURVEY Q7)
constexpr int32_t kVarFlagPadEdge = 2;      // fewer values than elements is not an error: the caller pads (B200TFS_OF_PAD_EDGE)

struct VarSeg {       // a contiguous run of one job: the whole tensor (encode) or one wire chunk (decode)
  const uint8_t* src;
  uint64_t n;         // elements (encode) or bytes (decode)
  uint32_t job;
  uint32_t first_tile;
};

constexpr uint32_t kVarGroupTiles = kVarThreads;  // tiles per counter group (one counter per thread when a CTA sums its prefix)

struct VarJobDev {
  uint8_t* dst;        // encode: first payload byte on the wire; decode: first element of the tensor
  uint64_t n_elems;
  uint64_t cap;        // encode: payload bytes the header announced (never written past)
  uint32_t* tile_val;  // [n_tiles] bytes (encode) / terminators (decode) of every tile of the job
  uint32_t* group_sum; // [ceil(n_tiles / kVarGroupTiles)] sums of tile_val; zeroed before the counting kernel
  unsigned long long* total;  // sum over the job; zeroed likewise
  int32_t* status;     // decode: B200TFS_OK or the first error
  int32_t dtype;       // DT_* of the tensor in memory
  uint32_t elem_size;
  uint32_t is_signed;
  int32_t flags;
  uint32_t first_tile;
  uint32_t n_tiles;
  uint32_t pad[2];
};

// what every varint kernel receives (by value, in the parameter space).  A single job with a single segment - one
// big tensor, the case where the bandwidth matters - travels inline, so that no CTA starts with three dependent loads.
struct VarTables {
  const VarSeg* segs;
  const uint32_t* tile_seg;
  const VarJobDev* jobs;
  uint32_t n_tiles;
  uint32_t single;      // 1: seg0 / job0 below describe every tile
  VarSeg seg0;
  VarJobDev job0;
  const uint32_t* n_tiles_dev;   // vdec_*_dev_kernel: the tile count vdec_plan_kernel left in device memory (n_tiles is then a bound)
};

// ---- packed-varint outputs of the single-launch decode (b200tfs_set_decode_varints) ----------------------------------
// vdec_plan_kernel reads the table the fused launch published and builds the decode tables on the device: output k of
// record r is job r * kFusedMaxOutputs + k and owns segments [job * B200TFS_MAX_RUNS, + n_runs) - fixed slots, so the
// plan needs no atomics and the host needs no copy of the table.  Every tile table is sized by the host from a bound it knows.
constexpr uint32_t kVarPlanThreads = 1024;
constexpr int32_t kVarSlotIdle = 1;       // status word of a slot the plan did not take (not a packed-varint output to decode)
struct VarPlan {
  const b200tfs_output* outs;      // the fused launch's table (pinned host memory, written by that launch)
  const int32_t* n_outs;
  const int32_t* rec_status;
  const uint8_t* w;                // wire arena
  const uint64_t* rec_off;         // n > kFusedInlineRecs: device copy; else off_inl
  uint64_t off_inl[kFusedInlineRecs];
  uint8_t* dst;
  uint64_t dst_stride;
  uint32_t n, tile_cap;
  VarJobDev* jobs;                 // [n * kFusedMaxOutputs]
  VarSeg* segs;                    // [n * kFusedMaxOutputs * B200TFS_MAX_RUNS]
  uint32_t* tile_seg;              // [tile_cap]
  uint32_t* tile_val;              // [tile_cap]
  uint32_t* group_sum;             // [tile_cap / kVarGroupTiles + n * kFusedMaxOutputs]
  unsigned long long* total;       // [n * kFusedMaxOutputs]
  int32_t* status;                 // [n * kFusedMaxOutputs]
  uint32_t* n_tiles;               // [1]
};
// tiles a record of `len` bytes can need: each of its <= kFusedMaxOutputs * B200TFS_MAX_RUNS chunks of L bytes spans at most
// ceil((L + 15) / kVarTileBytes) windows, and the chunks lie inside the record
constexpr uint64_t var_record_tile_bound(uint64_t len) { return len / kVarTileBytes + 2 + 2ull * kFusedMaxOutputs * B200TFS_MAX_RUNS; }

// ---- decode into one tensor per key, concatenated along axis 0 (b200tfs_decode_concat) -----------------------------
// concat_plan_kernel (one CTA) reads the parse kernel's table, matches the requested keys, scans every record's bytes into
// its offset inside the key's destination and writes (a) a move plan image - PlanHeader | MoveItem[n * n_keys *
// B200TFS_MAX_RUNS] (fixed slots) | TileRef[tile_cap] - that move_kernel runs over with a grid of tile_cap CTAs (the ones
// past PlanHeader::n_tiles leave at once), and (b) a table in the single-launch decode's layout (kFusedMaxOutputs slots per
// record, dst_off = the absolute destination address, dst_stride 0) that vdec_plan_kernel turns into packed-varint jobs.
constexpr uint32_t kConcatPlanThreads = 1024;
struct ConcatKeyDev { const uint8_t* key; uint8_t* dst; uint64_t cap; uint32_t key_len, pad; };
struct ConcatPlan {
  const uint8_t* w;                // wire arena
  const uint64_t* rec_off;         // [n], device
  const b200tfs_output* outs;      // parse table: record r at outs[r * out_stride]
  const int32_t* n_outs;
  const int32_t* rec_status;
  const ConcatKeyDev* keys;        // [n_keys]
  uint32_t n, n_keys, out_stride, cast;
  uint32_t vpt, tile_cap;
  int32_t* kst;                    // [n * n_keys] scratch: (record, key) status before the consistency checks
  int32_t* match;                  // [n * n_keys] scratch: table index of the key in the record, -1 if absent
  uint8_t* plan;                   // move plan image
  b200tfs_output* vouts;           // [n * kFusedMaxOutputs]
  int32_t* vn_outs;                // [n]
  int32_t* vrec_status;            // [n]
};
// move tiles a record of `len` bytes can need for n_keys distinct outputs: every run of n_out <= its wire bytes takes at
// most n_out / tile + 1 tiles, and a record holds at most B200TFS_MAX_RUNS runs per output
constexpr uint64_t concat_record_tile_bound(uint64_t len, uint64_t tile_bytes, uint32_t n_keys) {
  return len / tile_bytes + 1ull + (uint64_t)n_keys * B200TFS_MAX_RUNS;
}

// ---- DT_STRING keys of the concatenated decode as byte columns (b200tfs_decode_concat_strings) -------------------------
// concat_plan_strings_kernel scans 8 * n_strings of every (record, string key) into dst_off, the record's first offset entry.
// Then (string_kernels.cuh): str_index_kernel - a warp per pair walks its string_val elements (string_walk.h) and packs each
// one's record-relative wire offset (high 32 bits) and its byte position within the record's strings (low 32 bits) into the
// offset entry the string owns, and leaves the pair's byte total; str_scan_kernel - one CTA places every pair's bytes in the
// key's data and numbers the copy chunks (kStrChunk strings each); str_copy_kernel - a lane per short string, the warp for long
// ones; str_fix_kernel - the offsets' final values, in a launch of its own because the copy reads the entry behind each string.
constexpr uint32_t kStrChunk = 256;         // strings per copy chunk (eight per lane)
constexpr uint32_t kStrThreads = 256;       // threads per CTA of the index, copy and fix kernels
struct StrKeyDev { uint8_t* data; uint64_t cap; };
struct StrTables {
  const uint8_t* w;                // wire arena
  const uint64_t* rec_off;         // [n], device
  const uint64_t* rec_len;         // [n], device
  b200tfs_output* vouts;           // the plan's table: record r, key k at r * kFusedMaxOutputs + k (dst_off absolute)
  StrKeyDev keys[B200TFS_CONCAT_MAX_KEYS];   // the keys' string data (in the kernel parameters: a replay reads them as captured)
  uint64_t* bytes;                 // [n_keys * n]: the pair's string bytes (index)
  uint64_t* data0;                 // [n_keys * n]: its first byte in the key's data (scan)
  uint64_t* chunk0;                // [n_keys * n]: its first copy chunk (scan; key-major, so it rises through the array)
  uint64_t* n_chunks;              // [1]: chunks of every pair
  uint32_t n, n_keys;
};

// ---- decode into one padded tensor per key (b200tfs_decode_padded) ----------------------------------------------------
// padded_plan_kernel (one CTA) matches the keys as concat_plan_kernel does (plan_key_reference), checks every record against the
// first one that decoded the key and against the destination's trailing dims, scans the rows into first rows and writes one
// PadDesc per (record, key), the per-key summary and the single-launch decode's table for the varint tail (as ConcatPlan::vouts).
// padded_emit_kernel then writes the destination in chunks of kPadChunkBytes, a grid-stride loop over the chunks of every key.
constexpr uint32_t kPadEmitThreads = 256;
constexpr uint32_t kPadEmitVecs = 4;                                  // 16-byte vectors per thread and chunk
constexpr uint64_t kPadChunkBytes = 16ull * kPadEmitThreads * kPadEmitVecs;
struct PadKeyDev {
  ConcatKeyDev k;                  // key bytes, dst, cap
  int64_t dims[B200TFS_MAX_RANK];  // the destination's trailing dims (dims[0] unused)
  uint8_t pad[16];                 // the pad element's bits
  int32_t rank, pad_;
};
struct PadDesc {                   // one (record, key): its value runs, its own dims, its rows in the destination
  b200tfs_run runs[B200TFS_MAX_RUNS];
  int64_t dims[B200TFS_MAX_RANK];
  const uint8_t* rec;
  uint64_t first_row, rows;        // rows 0: no place
  uint32_t n_runs, pad_;
};
struct PadKeyOut {                 // one key after the plan
  uint64_t rows, pitch;            // rows in use, destination bytes per row
  uint64_t chunk0;                 // first chunk of the key (entry n_keys: the chunks of every key)
  uint32_t row_elems, esz, src_esz, op, varint, str;   // str: a DT_STRING key (padded_plan_strings_kernel), no chunks
};
struct PaddedPlan {
  ConcatPlan cp;                   // the parse table, scratch and varint table (cp.keys unused)
  const PadKeyDev* keys;           // [n_keys]
  PadDesc* desc;                   // [n * n_keys]: record r, key k at r * n_keys + k
  uint64_t* first_row;             // [n_keys * n]
  PadKeyOut* kout;                 // [n_keys + 1]
};
// the varint tail of the padded decode: job s = r * kFusedMaxOutputs + k (vdec_plan_kernel's slot) stores element e of record r
// at its padded position - mixed-radix over the record's dims into the destination's - from jb.dst, the record's first row
struct VarPadMap { const PadDesc* desc; const PadKeyDev* keys; uint32_t n_keys, pad_; };

// ---- DT_STRING keys of the padded decode as padded byte columns (b200tfs_decode_padded_strings) --------------------------
// padded_plan_strings_kernel places a string key's rows as any other key's, 8 bytes (one offset entry) per position.  Then
// (padded_kernels.cuh): pad_str_index_kernel - a warp per pair walks its string_val elements and packs
// each one's record-relative wire offset and byte position within the record's own strings into the offset entry of its padded
// position, and leaves the pair's own bytes; pad_str_scan_kernel - one CTA places every record's bytes (own strings plus pad_len
// per pad position) in the key's data, cuts the rows in use at the first record past data_cap and numbers the positions;
// pad_str_copy_kernel - destination-major, a lane per position: its own string or the pad, and the final offset of a pad position;
// pad_str_fix_kernel - the final offsets of the own strings, in a launch of its own because the copy reads those entries.
struct PadStrKeyDev { uint8_t* data; uint64_t cap; const uint8_t* pad; uint64_t pad_len; };
struct PadStrTables {
  PaddedPlan pp;                   // the plan's tables (PadKeyOut::rows of a string key: its rows in use, after the scan)
  const uint64_t* rec_len;         // [n], device
  PadStrKeyDev keys[B200TFS_CONCAT_MAX_KEYS];   // in the kernel parameters: a replay reads them as captured
  uint64_t* bytes;                 // [n_keys * n]: the pair's own string bytes (index)
  uint64_t* data0;                 // [n_keys * n]: its first byte in the key's data (scan)
  uint64_t* pos0;                  // [n_keys + 1]: the key's first position among the positions in use of every key (scan)
};

// ---- deferred framing: the length prefixes of packed-varint inputs computed ON THE DEVICE -----------------------------
// Every length on the wire precedes its content, and a packed-varint payload's length is only known once the counting
// kernel has run.  Instead of bringing it to the host (b200tfs_measure: a stream synchronise in the middle of an encode),
// the host uploads what each request's framing is made of - its model_spec bytes, and per input the key, the dims, the wire
// dtype and where the payload's length comes from - and frame_requests_kernel (one thread per request) runs the framing writers
// (framing.h write_request) over it: it counts the record, places it in its slot, writes the framing and patches the
// destinations into the move plan / the emit jobs that run right behind it.  No host round trip: the whole encode is
// asynchronous and CUDA-graph capturable.
constexpr uint32_t kTinyVarElems = 32;   // a packed-varint input of at most this many elements (a label, an id, a few flags) is
                                         // counted AND written by the framing kernel itself: no counting or emit kernel for it
struct TinyVar { const uint8_t* src; uint32_t n, elem_size, is_signed, pad; };
enum DeferredPayload : uint32_t {
  DP_NONE = 0,    // no payload
  DP_ITEM = 1,    // MoveItem idx moves it (dst patched)
  DP_SMALL = 2,   // SmallItem idx moves it (dst patched)
  DP_JOB = 3,     // varint job idx emits it: its length is totals[idx] (dst and cap patched)
  DP_TINY = 4     // TinyVar idx: the framing kernel counts and writes it
};
struct DeferredIn {         // one input of a request, in wire order
  uint64_t len;             // payload bytes of DP_ITEM / DP_SMALL
  uint32_t key_off, key_len;   // key bytes in FrameTables::blob
  uint32_t dims_off;        // int64 dims[rank] in FrameTables::blob
  int32_t rank, wire_dtype;
  uint32_t flags, field;
  uint32_t kind, idx;       // DeferredPayload and its index
  uint32_t pad;
};
struct DeferredReq {
  uint32_t spec_off, spec_len;   // the model_spec field (its tag included) in FrameTables::blob
  uint32_t grpc;                 // gRPC's five-byte length-prefixed-message header in front
  uint32_t first_in, n_in;
  uint32_t align_in;             // the input whose payload should start 128-byte aligned (request-local), ~0u: none
  uint32_t anchor_in;            // ~0u, or a DP_ITEM input whose first byte the host fixed at anchor_off: the record is laid out around it
  uint32_t tail_len;             // the output_filter run, in FrameTables::blob right behind the model_spec field
  uint64_t anchor_off;
  uint64_t slot_off, slot_cap;   // where the record may lie inside the arena (worst-case sized by the host)
};
struct FrameTables {
  const DeferredReq* reqs; const DeferredIn* ins; const uint8_t* blob;
  const unsigned long long* totals;   // packed length of every varint job (the counting kernel's result), by job index
  const TinyVar* tiny;                // DP_TINY
  uint8_t* arena;
  MoveItem* items; SmallItem* smalls; VarJobDev* jobs;    // patched
  uint64_t* rec_off; uint64_t* rec_len; int32_t* status;  // pinned host memory: read by b200tfs_encode_results
  uint32_t n;
};

// decode tiles of a chunk [src, src + n): aligned windows of kVarTileBytes starting at src rounded down to 16
B2_PLAN_HD uint64_t var_decode_tiles(const void* src, uint64_t n) {
  return n ? (((uint64_t)((uintptr_t)src & 15) + n + kVarTileBytes - 1) / kVarTileBytes) : 0;
}

// ---- tf.Example requests (example_host.inc plans, example_kernels.cuh runs) ----------------------------------------------
// One request's examples start at a host-fixed anchor inside its slot; the request prefix is written in front of them once
// their total is known.  Requests whose size depends on their values (an integer or a ragged column) get their example sizes
// from the count kernel and their offsets from the scan kernel (tiles of kExTile examples); the others have one closed-form
// example size.  A bytes column (EXO_BYTES, only in calls that run the kExColumns kernels) is counted like an integer one.
enum ExOp : uint32_t { EXO_F32 = 0, EXO_F64 = 1, EXO_F16 = 2, EXO_INT = 3, EXO_BOOL = 4, EXO_BYTES = 5 };
// which instantiation of the count and emit kernels a call runs: no variable-length column, a ragged numeric column, a bytes column
enum ExMode : int { kExDense = 0, kExRagged = 1, kExColumns = 2 };
constexpr uint32_t kExTile = kConcatPlanThreads;   // examples per count / scan CTA (one thread each in the scan)
constexpr uint32_t kExEmitThreads = 256;
constexpr uint32_t kExStage = 16384;               // shared-memory image of the wire one emit batch writes
struct ExFeat {             // one column of one request, in wire order
  const uint8_t* data;
  uint64_t row_stride;      // bytes between the rows of consecutive examples (0: a broadcast column)
  uint64_t row_elems;
  uint32_t op, esz, sgn;    // ExOp, element size in memory, sign-extend (EXO_INT)
  uint32_t key_off, key_len;   // key bytes in ExTables::blob
  uint32_t lcol;            // integer columns: column of the request's length table
  const int64_t* lengths;   // a ragged column: example i takes min(max(lengths[i], 0), max_len) * unit elements; NULL: dense
  uint64_t max_len, unit;   // row_elems == max_len * unit
  const int64_t* offsets;   // EXO_BYTES: string j is data[offsets[j], offsets[j+1]); example i's row starts at string i * row_stride
  uint64_t data_len;        // (row_stride = row_elems, or 0 for a broadcast column).  Last: the dense and ragged kernels never read them
};
// The prefix the frame kernel writes in front of the examples, for both targets:
//   [00 be32(msg)] spec 12 vi(outer) mid inner_tag vi(inner) head | examples [output_filter run: Predict only]
//   example_list (Classify / Regress):  outer = Input, mid and head empty, inner_tag 0A, inner = ExampleList
//   Predict string_val:                 outer = the inputs map entry, mid = 0A vi(klen) key, inner_tag 12, inner = TensorProto,
//                                       head = 08 07 12 vi(shape) {tensor_shape: dim {size: n}}
struct ExReq {
  uint32_t first_feat, n_feat, n_int;   // integer columns (their entries per example in ExTables::L)
  uint32_t spec_off, spec_len;          // the model_spec field (tag included) in ExTables::blob, followed there by mid and head
  uint32_t grpc;                        // gRPC's five-byte length-prefixed-message header in front
  uint32_t first_tile, n_tiles;         // count / scan tiles (requests whose size depends on their values)
  uint64_t n_ex, ex0;                   // examples, and the first one's index in the per-example tables of the call
  uint64_t L0;                          // first entry of the request in ExTables::L (n_ex * n_int entries)
  uint64_t fixed_size;                  // bytes of every example in the example_list (its tag included); 0: the size depends on
                                        // the values (an integer or a ragged column), S and off hold each example's
  uint64_t anchor, slot_end;            // arena offsets: where example 0 starts, where the slot ends
  uint32_t mid_len, head_len, inner_tag;        // the Predict prefix above (example_list: 0, 0, 0A); last, because among the
                                                // fields the emit kernel reads they cost ex_emit_kernel<false> 12 registers
  uint32_t n_ctx;                               // a SequenceExample request: its first n_ctx features (wire order) are context
  uint32_t tail_len, pad_;                      // a Predict form's output_filter run, in ExTables::blob behind head, written
                                                // behind the examples (and the context) by the frame kernel
};
struct ExSpan { uint32_t req, pad; uint64_t e0, e1; };   // a CTA's examples [e0, e1) of request `req`
// A call with contexts (ExampleListWithContext) plans each present context as one more request entry of one example, at an
// index >= n_req of ExTables::reqs: its features, L entries and count tile are its own (an empty context: no feature, no tile,
// fixed_size 2, the bytes 12 00).  The frame kernel writes it behind the request's examples, behind the tag 12:
//   [00 be32(msg)] spec 12 vi(outer) mid 12 vi(inner) head [42 vi(elwc)] | examples... | 12 vi(ctx) 0A vi(F) entries
// with the ELWC nested in a string_val (`nest`) in the Predict form.  One entry per request of the call.
constexpr uint32_t kExNoContext = 0xFFFFFFFFu;
struct ExCtxRef { uint32_t req, nest; };   // the context's entry in ExTables::reqs (kExNoContext: none), Predict-ELWC
// A batch of ExampleListWithContexts (PREDICT_ELWCS, one per query) is a request entry over all its examples, whose emit spans
// never cross a query, and one context entry of Q "examples" over the context columns, one span each.  Both are scanned
// contiguously; query q then moves by a shift that opens the gaps for the headers and contexts in front of it:
//   ... 12 vi(inner) head | {42 vi(E_q + C_q) | query q's examples (E_q bytes) | 12 vi(ctx) context q (C_q bytes)}*
// ex_frame_lists_kernel computes every shift, writes the headers (and the 12 00 of empty contexts) before the emits run.  The
// request's ExCtxRef is {its index into ExLists::lists, kExListRef}.
constexpr uint32_t kExListRef = 2;
struct ExList { uint32_t req, ctx, q0, n_q; };   // the request entry, its context entry, its queries [q0, q0 + n_q)
struct ExQuery { uint64_t e0, e1; };              // a query's examples [e0, e1) of its request
struct ExLists {
  const ExList* lists; const ExQuery* queries;
  uint64_t* shift;                      // per query: arena offset from the anchor minus the contiguous offset, of its examples
  uint64_t* cshift;                     // and of its context
  uint32_t n_lists, n_spans, n_ctx_spans, pad_;   // emit spans behind all others: the examples', then one per non-empty context
};
// A PREDICT_ELWCS request whose list sizes are in device memory (b200tfs_example_device_lists) has no ExQuery entries and no
// host-cut spans: ex_frame_lists_dev_kernel scans its sizes into query ranges, clamped into [0, n_ex] (a negative size or an
// overflow makes the request B200TFS_E_SHAPE), and writes its example spans into n_s scratch slots from s0, cut every `per`
// examples and at every query's end.  A query adds at most one partial span, so n_s = ceil(n_ex / per) + Q always holds them;
// the unused slots are empty (e1 == e0), which ex_emit_list_dev_kernel leaves at once.  Its queries' shifts follow those of all
// host-sized queries (ExList::q0 indexes ExLists::shift / cshift only).  One entry per ExLists::lists entry; sizes NULL: host.
struct ExListSizes { const int64_t* sizes; uint64_t per; uint32_t s0, n_s; };
struct ExDevLists {
  const ExListSizes* lists;
  ExSpan* spans;                        // scratch: the example spans of the device-sized requests, behind each other
  uint32_t n_spans, pad_;
};
struct ExTables {
  const ExReq* reqs; const ExFeat* feats; const uint8_t* blob;
  const ExSpan* tiles;                  // count / scan CTAs
  const ExSpan* spans;                  // emit CTAs: those of the example_list requests, then the n_predict_spans of the Predict ones
  uint64_t* L;                          // packed length of every (example, integer column), or list length (bytes column)
  uint64_t* S;                          // bytes of every example of a request whose size depends on its values
  uint64_t* off;                        // its offset from the anchor
  unsigned long long* tile_sum;         // bytes of every tile's examples
  int32_t* bad;                         // a call with a ragged or bytes column: per request (and context entry), nonzero when a
                                        // length or a string offset was out of range (zeroed by the host in every call); NULL
                                        // otherwise
  uint8_t* arena;
  uint64_t* rec_off; uint64_t* rec_len; int32_t* status;   // pinned host memory: read by b200tfs_encode_results
  uint32_t n_req, n_tiles, n_spans, n_predict_spans;
};
// Bytes of one feature map entry (its tag included) whose list payload is P bytes; *hl receives those in front of the payload:
//   0A vi(entry) 0A vi(klen) key 12 vi(Feature) {12 float_list | 1A int64_list} vi(list) [0A vi(P) payload]
B2_PLAN_HD uint64_t ex_entry_len(uint64_t P, uint64_t klen, uint64_t* hl) {
  const uint64_t list = P ? 1 + varint_len(P) + P : 0, feature = 1 + varint_len(list) + list;
  const uint64_t entry = 1 + varint_len(klen) + klen + 1 + varint_len(feature) + feature;
  *hl = 1 + varint_len(entry) + entry - P;
  return 1 + varint_len(entry) + entry;
}
// The same for a bytes_list, whose repeated strings are not packed: its list is the P bytes of {0A vi(len) bytes} fields.
//   0A vi(entry) 0A vi(klen) key 12 vi(Feature) 0A vi(P) {0A vi(len) bytes}*
B2_PLAN_HD uint64_t ex_bytes_entry_len(uint64_t P, uint64_t klen, uint64_t* hl) {
  const uint64_t feature = 1 + varint_len(P) + P;
  const uint64_t entry = 1 + varint_len(klen) + klen + 1 + varint_len(feature) + feature;
  *hl = 1 + varint_len(entry) + entry - P;
  return 1 + varint_len(entry) + entry;
}
// bytes of one example in the example_list or string_val (its tag included) whose map entries add up to F bytes:
// {0A | 42} vi(X) 0A vi(F) entries
B2_PLAN_HD uint64_t ex_example_len(uint64_t F) {
  const uint64_t x = 1 + varint_len(F) + F;
  return 1 + varint_len(x) + x;
}

// the most bytes of one query's 42 vi(E + C) header (E + C < 2 GiB)
constexpr uint64_t kExListHeader = 6;

// ---- SequenceExamples (PREDICT_SEQUENCE requests; ex_seq_count_kernel, ex_emit_sequence_kernel) -------------------------
// A sequence request is one ExReq whose features [0, n_ctx) are context features (an example's, in wire order) and the rest
// feature lists, each an ExFeat with max_len = T steps of `unit` elements (row_elems = T * unit; lengths: sequence i has
// min(max(lengths[i], 0), T) steps, NULL: T).  An integer or bytes list takes T columns of ExTables::L from lcol on, one per step:
// the step's list payload.  Sequence requests are always counted; their count tiles and emit spans follow all the others.
//   42 vi(S) 0A vi(C) {context map entries} 12 vi(G) {0A vi(e) 0A vi(klen) key 12 vi(FL) {0A vi(feat) Feature}*}*
// One step (its 0A tag included) whose Feature holds a list of payload P (bytes: P bytes of {0A vi(len) bytes} fields)
B2_PLAN_HD uint64_t sq_step_len(uint64_t P, bool bytes) {
  const uint64_t list = bytes ? P : P ? 1 + varint_len(P) + P : 0, feature = 1 + varint_len(list) + list;
  return 1 + varint_len(feature) + feature;
}
// the FeatureLists map entry (its tag included) of a list whose steps take FL bytes
B2_PLAN_HD uint64_t sq_list_entry_len(uint64_t FL, uint64_t klen) {
  const uint64_t e = 1 + varint_len(klen) + klen + 1 + varint_len(FL) + FL;
  return 1 + varint_len(e) + e;
}
// a sequence in the string_val (tag 42 included) whose context entries take C bytes and list entries G
B2_PLAN_HD uint64_t sq_sequence_len(uint64_t C, uint64_t G) {
  const uint64_t x = 1 + varint_len(C) + C + 1 + varint_len(G) + G;
  return 1 + varint_len(x) + x;
}

// ---- Classify / Regress responses (example_host.inc plans, example_resp_kernels.cuh runs) --------------------------------
// Every buffer is sized from the record lengths alone: response r owns xr_row_bound(rec_len[r]) entry slots from ent0[r] on.
constexpr uint32_t kXrIndexWarps = 4;      // responses per index CTA (one warp each)
constexpr uint32_t kXrEmitThreads = 128;   // emit: one thread per row (a Regression entry or a Classifications example)
struct XrTables {
  const uint8_t* w;                        // the arena
  const uint64_t* rec_off; const uint64_t* rec_len; const uint64_t* ent0;
  b200tfs_label_ref* ent;                  // {off, len} of every result entry, record-relative
  uint32_t* rows;                          // entries of every response
  uint32_t* cls0;                          // Classify: classes of every response's first example
  int32_t* status;                         // B200TFS_OK / E_PARSE / E_SIZE / E_SHAPE (lowest wins)
  b200tfs_model_spec* specs;
  uint64_t* row0;                          // first row of every response (scan)
  unsigned long long* batch;               // rows, C, first response with rows, same_labels
  float* values; uint64_t values_cap;
  b200tfs_label_ref* labels; uint64_t labels_cap;
  int64_t* per_rec_host; b200tfs_model_spec* specs_host; int64_t* batch_host;   // pinned host memory: read by b200tfs_example_response_results
  uint32_t n, kind;
};

// ---- MultiInference responses (example_host.inc plans, multi_resp_kernels.cuh runs) ---------------------------------------
// Response r owns xr_row_bound(rec_len[r]) entry slots from E0[r] on, shared by its tasks: task t's entries follow task t - 1's.
// The per-task tables are task-major, [n_tasks][n]; task t's XrTables view points at its rows, and the xr kernels run on it.
struct MiTables {
  const uint8_t* w;
  const uint64_t* rec_off; const uint64_t* rec_len; const uint64_t* E0;
  const uint32_t* kinds;                   // B200TFS_RESP_* of every task
  b200tfs_label_ref* ent;
  uint64_t* ent0; uint32_t* rows; uint32_t* cls0; int32_t* status; b200tfs_model_spec* specs;   // [n_tasks][n]
  uint32_t n, n_tasks;
};

}  // namespace b200tfs
