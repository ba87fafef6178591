/* b200tfs.h - C ABI of libb200tfs.so: the TensorProto / PredictRequest / PredictResponse wire codec
 * of zendesk/min-tfs-client's Predict hot path, run as hand-written sm_90a (H100) CUDA kernels.
 *
 * The reference has no FFI: its hot path is Python calling the protobuf runtime.  The seams this
 * library replaces are (paths relative to the reference checkout):
 *
 *   encode   tensor_serving_client/min_tfs_client/tensors.py:28-35   ndarray_to_tensor_proto
 *            tensor_serving_client/min_tfs_client/tensors.py:17-25   write_values_to_tensor_proto
 *            tensor_serving_client/min_tfs_client/requests.py:41-48  PredictRequest assembly
 *            protobuf_srcs/tensorflow_serving/apis/prediction_service_pb2_grpc.py:52
 *                                                                     PredictRequest.SerializeToString
 *   decode   protobuf_srcs/tensorflow_serving/apis/prediction_service_pb2_grpc.py:53
 *                                                                     PredictResponse.FromString
 *            tensor_serving_client/min_tfs_client/tensors.py:38-46   extract_shape, tensor_proto_to_ndarray
 *   dtypes   tensor_serving_client/min_tfs_client/constants.py:13-29 numpy <-> DT_* <-> TensorProto field
 *
 * Plain C: pointers, sizes, int status codes.  No torch / numpy / protobuf types cross this line.
 * Every function returns B200TFS_OK (0) or a negative B200TFS_E_* code; b200tfs_last_error() gives
 * the thread-local message.  Nothing here ever falls back to a CPU codec: without a CUDA device
 * b200tfs_create() fails with B200TFS_E_CUDA and every codec entry point needs a context.
 *
 * Threading: a b200tfs_ctx owns pinned/device scratch plus a CUDA stream (or borrows the caller's: b200tfs_set_stream) and is
 * NOT re-entrant; use one context per calling thread (contexts are cheap).  Distinct contexts are independent.
 */
#ifndef B200TFS_H_
#define B200TFS_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200TFS_ABI_VERSION 2

/* ---- status codes ---------------------------------------------------------------------------- */
#define B200TFS_OK 0
#define B200TFS_E_DTYPE (-1)        /* dtype not in the reference's table / cast not supported   (ValueError) */
#define B200TFS_E_SHAPE (-2)        /* bad rank / dims / element count != prod(shape)            (ValueError) */
#define B200TFS_E_SIZE (-3)         /* caller buffer too small                                                */
#define B200TFS_E_PARSE (-4)        /* malformed protobuf wire                                   (DecodeError) */
#define B200TFS_E_CUDA (-5)         /* CUDA runtime error / no device                                          */
#define B200TFS_E_TOOBIG (-6)       /* message would exceed protobuf's 2 GiB limit                            */
#define B200TFS_E_ARG (-7)          /* bad argument                                                            */
#define B200TFS_E_NONCANONICAL (-8) /* valid wire, but a layout this entry point does not tabulate (the single-launch
                                       decode: values in more runs / more dims than the table holds inline; both
                                       parsers: groups or variant tensors nested deeper than 16)                     */
#define B200TFS_E_RANGE (-9)        /* decoded integer does not fit the target dtype          (OverflowError) */
#define B200TFS_E_KEY (-10)         /* dtype enum absent / unmapped on decode                       (KeyError) */
#define B200TFS_E_SPILL (-11)       /* internal to the parsers: a record needs a larger spill area (the two-phase parse
                                       grows it and runs again; callers never see this code)                        */

/* ---- tensorflow.DataType values used on this path (types.proto:12-68; pinned by the reference's
 *      tests/unit/min_tfs_client/types_test.py:7-23) ------------------------------------------------ */
#define B200TFS_DT_INVALID 0
#define B200TFS_DT_FLOAT 1
#define B200TFS_DT_DOUBLE 2
#define B200TFS_DT_INT32 3
#define B200TFS_DT_UINT8 4
#define B200TFS_DT_INT16 5
#define B200TFS_DT_INT8 6
#define B200TFS_DT_STRING 7
#define B200TFS_DT_COMPLEX64 8
#define B200TFS_DT_INT64 9
#define B200TFS_DT_BOOL 10
#define B200TFS_DT_BFLOAT16 14 /* not in the reference's table; TF convention (half_val bit patterns) */
#define B200TFS_DT_UINT16 17
#define B200TFS_DT_COMPLEX128 18
#define B200TFS_DT_HALF 19
#define B200TFS_DT_UINT32 22
#define B200TFS_DT_UINT64 23
/* unpack-only pseudo dtype: decode DT_HALF the way the reference does - half_val integers taken as
 * VALUES and converted to float16 (18688 -> 18688.0), SURVEY 8a Q7 - instead of TF's bit patterns */
#define B200TFS_DT_HALF_REFQUIRK (-19)

/* ---- encode flags (b200tfs_tensor.flags) ------------------------------------------------------- */
#define B200TFS_F_TENSOR_CONTENT 0x1u /* emit raw little-endian bytes in tensor_content (field 4) instead of the
                                         typed repeated field the reference writes (tensors.py:17-25)            */
#define B200TFS_F_KEEP_SNAN 0x2u      /* do NOT quiet float32 signalling NaNs.  Default quiets them, because the
                                         reference routes every float32 through a Python double (tensors.py:22). */
#define B200TFS_F_PRESERIALIZED 0x4u  /* `data` already holds a serialised TensorProto of `packed_len` bytes (how the
                                         host hands over DT_STRING tensors, tensors.py:24): spliced in verbatim        */
#define B200TFS_F_DEVICE_DATA 0x8u    /* *_host entry points only: `data` of THIS tensor is a device pointer already (a tensor
                                         that lives in HBM - the usual case for a model's activations): it is not staged      */

/* ---- decode flags (b200tfs_output.flags, set by the parser) ----------------------------------- */
#define B200TFS_OF_TENSOR_CONTENT 0x1u /* values arrived in tensor_content                                        */
#define B200TFS_OF_MULTI_CHUNK 0x2u    /* values field split over several occurrences / unpacked elements         */
#define B200TFS_OF_UNPACKED 0x80u      /* some values arrived as unpacked scalar elements (wire type 0 / 1 / 5)   */
#define B200TFS_OF_SPILLED 0x100u      /* more dims than B200TFS_MAX_RANK and / or more value runs than B200TFS_MAX_RUNS: the rest
                                          is held by the context (b200tfs_output_dims / b200tfs_output_runs)               */
#define B200TFS_OF_DIM_INFERRED 0x4u   /* one dim was -1 and was inferred from the element count                 */
#define B200TFS_OF_HAS_UNKNOWN 0x8u    /* unknown fields were skipped inside this entry                           */
#define B200TFS_OF_RANK0 0x10u         /* no dims: the reference raises TypeError here (reshape() with no args)   */
#define B200TFS_OF_VARINT 0x20u        /* values are packed varints: element count is checked while unpacking    */
#define B200TFS_OF_PAD_EDGE 0x40u      /* set by the CALLER of b200tfs_unpack_outputs on an output tabulated with
                                          B200TFS_E_SHAPE (or on any B200TFS_OF_VARINT output, whose element count only the
                                          decode kernels learn): TensorFlow's MakeNdarray convention (tensor_util.py:636-642 in
                                          the reference's vendored tree) - fewer values than the shape holds: the last one
                                          repeats; no values at all: zeros.  More values than the shape holds stays an error */

/* map-entry order for requests with several inputs (SURVEY 8a Q1) */
#define B200TFS_ORDER_GIVEN 0 /* emit in the order of b200tfs_request.inputs                                     */
#define B200TFS_ORDER_UPB 1   /* the order SerializeToString(deterministic=True) gives with the protobuf (upb)
                                 runtime the oracle was pinned against: bytewise, but a key that is a strict prefix
                                 of another sorts AFTER it                                                          */
/* b200tfs_request.flags */
#define B200TFS_RF_GRPC_FRAME 0x1 /* put gRPC's length-prefixed-message header in front of the record: one byte 0 (not
                                     compressed) and the message length as a big-endian uint32 (what grpc writes on the HTTP/2
                                     stream before the bytes request_serializer returned); rec_off/rec_len and
                                     b200tfs_request_size include the five bytes                                          */
#define B200TFS_ORDER_BYTES 2 /* plain bytewise order (shorter prefix first)                                     */

#define B200TFS_MAX_RANK 16   /* dims held inline by b200tfs_output; deeper shapes spill (b200tfs_output_dims).  Encode
                                 accepts any rank up to 254 (TF's limit)                                          */
#define B200TFS_MAX_RUNS 8    /* value runs held inline by b200tfs_output; more spill (b200tfs_output_runs)      */

typedef struct b200tfs_ctx b200tfs_ctx;

/* One tensor to encode.  `data` is a DEVICE pointer for b200tfs_encode_* and a HOST pointer for the
 * *_host variants; elements are C-contiguous, little-endian, in `src_dtype`.  `wire_dtype` is the
 * DT_* written into the TensorProto; if it differs from src_dtype the kernel casts while packing
 * (HALF->FLOAT and BFLOAT16->FLOAT, both exact; see b200tfs_cast_supported()).                   */
typedef struct b200tfs_tensor {
  const void* data;
  int32_t src_dtype;
  int32_t wire_dtype;
  int32_t rank;
  uint32_t flags;       /* B200TFS_F_*                                                        */
  const int64_t* dims;  /* rank entries                                                       */
  const char* key;      /* map key bytes (UTF-8, not NUL terminated); ignored for bare protos */
  int64_t key_len;
  uint64_t packed_len;  /* varint dtypes: byte length of the packed payload; filled by
                           b200tfs_measure(); ignored (recomputed) for fixed-width dtypes     */
} b200tfs_tensor;

/* One PredictRequest (predict.proto:12-27; assembled as reference requests.py:41-48 does). */
typedef struct b200tfs_request {
  const char* model_name;
  int64_t model_name_len;
  int32_t has_version;  /* model_version is not None (requests.py:44)                          */
  int32_t order;        /* B200TFS_ORDER_*                                                     */
  int64_t version;
  int32_t n_inputs;
  int32_t flags;        /* B200TFS_RF_*                                                        */
  const b200tfs_tensor* inputs;
} b200tfs_request;

/* Where the values of one output lie on the wire.  The reference iterates the merged repeated field whatever
 * its wire layout (tensors.py:42-46): one packed occurrence, several of them, single unpacked elements, or any
 * mix.  A run is `count` pieces of `len` value bytes each, `stride` bytes apart - one packed occurrence is a run
 * of count 1; a row of unpacked elements (tag + 4 value bytes, tag + 4 value bytes, ...) is ONE run of count n,
 * len 4, stride 5; equally long packed occurrences at equal distances coalesce the same way.                    */
typedef struct b200tfs_run {
  uint64_t off;    /* first piece, byte offset from the start of the record                    */
  uint32_t len;    /* value bytes per piece                                                     */
  uint32_t count;  /* pieces                                                                    */
  uint32_t stride; /* distance between the starts of consecutive pieces (0 when count == 1)    */
  uint32_t field;  /* TensorProto field number the pieces belong to                             */
} b200tfs_run;

/* One decoded output of a PredictResponse (predict.proto:30-40), as tabulated by the parse kernel.
 * All offsets are byte offsets from the start of the RECORD (arena + rec_off[i]).                  */
typedef struct b200tfs_output {
  uint64_t key_off;    /* map key bytes (last `key` occurrence of the winning entry)            */
  uint32_t key_len;
  int32_t dtype;       /* DT_* (last occurrence wins; 0 if absent)                              */
  int32_t rank;
  uint32_t flags;      /* B200TFS_OF_*                                                          */
  int32_t value_field; /* TensorProto field the dtype maps to (constants.py:13-29), 0 = unmapped */
  int32_t n_runs;      /* value runs of that field, in wire order (ALL of them; the first
                          B200TFS_MAX_RUNS are in runs[], see B200TFS_OF_SPILLED)                */
  int64_t dims[B200TFS_MAX_RANK];          /* after -1 inference; `rank` counts ALL dims        */
  b200tfs_run runs[B200TFS_MAX_RUNS];
  uint64_t content_off; /* tensor_content (field 4), last occurrence; content_len 0 if absent   */
  uint64_t content_len;
  uint64_t msg_off;     /* the TensorProto sub-message itself (last `value` occurrence)         */
  uint64_t msg_len;
  uint64_t n_elems;     /* prod(dims)                                                           */
  uint64_t dst_bytes;   /* n_elems * element size of `dtype` in memory                          */
  uint64_t n_strings;   /* string_val occurrences (strings are unpacked on the host)            */
  uint64_t dst_off;     /* b200tfs_decode_responses: where the values were written, from the
                           record's destination slot dst_dev + i*dst_stride                    */
  int32_t status;       /* B200TFS_OK, or the error tensor_proto_to_ndarray raises for it       */
  uint32_t n_inline;    /* entries of runs[] in use (== n_runs unless B200TFS_OF_SPILLED)        */
  uint32_t spill_rec;   /* B200TFS_OF_SPILLED: record index within the parse call and ordinal of the map   */
  uint32_t spill_seq;   /* entry inside it whose spill entries complete this output (opaque)     */
} b200tfs_output;

typedef struct b200tfs_model_spec {
  uint64_t name_off;  /* offsets from the start of the record                                  */
  uint32_t name_len;
  uint32_t signature_len;
  uint64_t signature_off;
  uint64_t label_off;
  uint32_t label_len;
  int32_t has_version;
  int64_t version;
} b200tfs_model_spec;

/* ---- library / context ----------------------------------------------------------------------- */
int b200tfs_abi_version(void);
const char* b200tfs_last_error(void);
int b200tfs_device_count(int* count);
int b200tfs_create(int device, b200tfs_ctx** out);
int b200tfs_destroy(b200tfs_ctx* ctx);
int b200tfs_sync(b200tfs_ctx* ctx);
void* b200tfs_stream(b200tfs_ctx* ctx); /* the cudaStream_t every call on this context is ordered on */
/* Order every LATER call of this context on the caller's stream (a cudaStream_t of the context's device; NULL: back to the
 * context's own stream).  Work already queued is ordered ahead of it by an event edge - nothing synchronises.  The stream
 * stays the caller's: it must outlive its use here and is not destroyed with the context.  Not during graph capture.     */
int b200tfs_set_stream(b200tfs_ctx* ctx, void* stream);
int b200tfs_kernel_launches(b200tfs_ctx* ctx, uint64_t* count); /* kernels launched so far on this context */

/* ---- memory + timing helpers so a ctypes host needs nothing but this library ------------------- */
int b200tfs_malloc(b200tfs_ctx* ctx, uint64_t bytes, void** dptr);
int b200tfs_free(b200tfs_ctx* ctx, void* dptr);
int b200tfs_host_alloc(uint64_t bytes, void** hptr); /* pinned */
int b200tfs_host_free(void* hptr);
int b200tfs_memcpy_h2d(b200tfs_ctx* ctx, void* dst_dev, const void* src_host, uint64_t bytes); /* async */
int b200tfs_memcpy_d2h(b200tfs_ctx* ctx, void* dst_host, const void* src_dev, uint64_t bytes); /* async */
int b200tfs_memcpy_d2d(b200tfs_ctx* ctx, void* dst_dev, const void* src_dev, uint64_t bytes);  /* async */
int b200tfs_memset(b200tfs_ctx* ctx, void* dst_dev, int value, uint64_t bytes);                /* async */
int b200tfs_event_create(void** ev);
int b200tfs_event_destroy(void* ev);
int b200tfs_event_record(b200tfs_ctx* ctx, void* ev);
int b200tfs_event_sync(void* ev);
int b200tfs_event_elapsed_ms(void* start, void* stop, float* ms);

/* ---- dtype table (constants.py:13-29, types.py:19-42) ------------------------------------------ */
/* element size in memory of a DT_* (0 if not a fixed-size numeric dtype on this path)            */
int b200tfs_dtype_size(int32_t dtype);
/* TensorProto field number the reference stores this dtype in (5 float_val, 6 double_val, 7 int_val,
 * 8 string_val, 9 scomplex_val, 10 int64_val, 11 bool_val, 12 dcomplex_val, 13 half_val, 16 uint32_val,
 * 17 uint64_val); 0 if unmapped                                                                    */
int b200tfs_dtype_field(int32_t dtype);
/* 1 if the encoder can read src_dtype memory and emit wire_dtype                                   */
int b200tfs_cast_supported(int32_t src_dtype, int32_t wire_dtype);

/* ---- sizes (host, closed form) ----------------------------------------------------------------- */
/* TensorProto for one tensor: header_len = bytes before the payload, total_len = whole message.
 * Varint dtypes need tensor->packed_len (see b200tfs_measure).                                     */
int b200tfs_tensor_proto_size(const b200tfs_tensor* t, uint64_t* header_len, uint64_t* total_len);
int b200tfs_request_size(const b200tfs_request* r, uint64_t* total_len);
/* The non-payload bytes, computed on the host exactly as the kernels will write them: the header of
 * one TensorProto (08 dtype 12 shape [values tag + length]) ...                                     */
int b200tfs_tensor_proto_header(const b200tfs_tensor* t, void* buf, uint64_t cap, uint64_t* len);
/* ... and every framing byte of a PredictRequest, concatenated in wire order, with - per input in
 * emission order - where its payload starts in the final message (payload_off), how long it is
 * (payload_len) and which inputs[] index it is (perm).  Needs no device.                           */
int b200tfs_request_frame(const b200tfs_request* r, void* buf, uint64_t cap, uint64_t* frame_len,
                          uint64_t* payload_off, uint64_t* payload_len, int32_t* perm);
/* Order the inputs of a request the way `order` says; writes a permutation of 0..n-1.              */
int b200tfs_order_keys(int32_t n, const char* const* keys, const int64_t* key_lens, int32_t order,
                       int32_t* perm);
/* Arena bytes needed to encode these records with b200tfs_encode_* (records are placed so that the
 * largest payload of each lands 128-byte aligned; the arena base must be 256-byte aligned).  A batch of requests in
 * which some packed-varint input has packed_len == 0 (not measured) is sized for b200tfs_encode_requests_async: one
 * worst-case slot per record.                                                                       */
int b200tfs_tensor_arena_size(int32_t n, const b200tfs_tensor* tensors, uint64_t* bytes);
int b200tfs_request_arena_size(int32_t n, const b200tfs_request* reqs, uint64_t* bytes);

/* ---- encode (device tensors -> device wire arena) ---------------------------------------------- */
/* Pass 1 for the varint-packed dtypes (int_val / int64_val / uint32_val / uint64_val / half_val):
 * fills tensors[i].packed_len on the device and copies the lengths back (synchronises).  The tensor's
 * contents must not change between this call and the encode that uses packed_len (the header announces
 * that length; the encoder never writes past it, but the bytes would be meaningless).  The per-tile
 * counters of the measurement stay on the device, keyed by tensors[i].data, and the NEXT encode of that
 * buffer on this context consumes them instead of counting again; any later encode counts afresh.     */
int b200tfs_measure(b200tfs_ctx* ctx, int32_t n, b200tfs_tensor* tensors);
/* n bare TensorProtos (what ndarray_to_tensor_proto(...).SerializeToString() returns).
 * rec_off/rec_len (host arrays of n) receive where each message lies inside the arena.  Async.     */
int b200tfs_encode_tensor_protos(b200tfs_ctx* ctx, int32_t n, const b200tfs_tensor* tensors,
                                 void* arena_dev, uint64_t arena_cap, uint64_t* rec_off,
                                 uint64_t* rec_len);
/* n PredictRequests (what PredictRequest.SerializeToString() returns for the request the reference
 * builds in requests.py:41-48).  Async.                                                            */
int b200tfs_encode_requests(b200tfs_ctx* ctx, int32_t n, const b200tfs_request* reqs, void* arena_dev,
                            uint64_t arena_cap, uint64_t* rec_off, uint64_t* rec_len);

/* The same encode (requests.py:41-48 + PredictRequest.SerializeToString, prediction_service_pb2_grpc.py:52) WITHOUT the host-side
 * measuring pass: inputs of the packed-varint dtypes (constants.py:16-23: int_val, int64_val, ...) may carry packed_len == 0.
 * Their lengths are counted, the length prefixes (and every length that encloses them) written, and the record placed by
 * kernels alone - count -> frame_requests_kernel (one thread per request evaluates the dependent varints, writes the
 * framing, patches the destinations of the payload movers) -> move + emit - so the call never synchronises and can be
 * captured in a CUDA graph (b200tfs_measure cannot).  Every record gets a 256-byte aligned slot sized for its worst case
 * (b200tfs_request_arena_size does that when it sees an unmeasured input) and lies inside it with its largest payload
 * 128-byte aligned; WHERE exactly, and how long it is, is known once the kernels have run: b200tfs_encode_results
 * synchronises and delivers rec_off / rec_len (or the first per-request error).  Bytes identical to b200tfs_encode_requests. */
int b200tfs_encode_requests_async(b200tfs_ctx* ctx, int32_t n, const b200tfs_request* reqs, void* arena_dev,
                                  uint64_t arena_cap);
int b200tfs_encode_results(b200tfs_ctx* ctx, int32_t n, uint64_t* rec_off, uint64_t* rec_len);
/* What frame_requests_kernel computes for ONE request, run on the host (the same inline code; needs no device): given the
 * packed length of every packed-varint input (packed_len[i] for inputs[i]; other entries ignored) it writes every framing
 * byte of the record into buf at the place it has on the wire and reports where the record lies (rec_off / rec_len) and,
 * per input, where its payload belongs (payload_off[i] / payload_len[i]; 0 / 0 for an input without values).            */
int b200tfs_request_frame_deferred(const b200tfs_request* r, const uint64_t* packed_len, void* buf, uint64_t cap,
                                   uint64_t* rec_off, uint64_t* rec_len, uint64_t* payload_off, uint64_t* payload_len);

/* ---- decode (device wire arena -> table -> device tensors) -------------------------------------- */
/* Parse n PredictResponse messages lying at rec_off[i]..+rec_len[i] of the device arena.  Runs the
 * parse kernel, then copies the table back (synchronises).  outs has n*max_outputs slots (record i
 * uses outs[i*max_outputs ...]); n_outs[i] receives the number of distinct keys; specs[i] the
 * model_spec.  rec_status[i] is B200TFS_OK or the error for that record.  Returns B200TFS_OK if the
 * kernel ran, even when individual records carry errors.                                           */
int b200tfs_parse_responses(b200tfs_ctx* ctx, const void* arena_dev, int32_t n, const uint64_t* rec_off,
                            const uint64_t* rec_len, int32_t max_outputs, b200tfs_output* outs,
                            int32_t* n_outs, b200tfs_model_spec* specs, int32_t* rec_status);
/* A shape deeper than B200TFS_MAX_RANK or values in more than B200TFS_MAX_RUNS runs (B200TFS_OF_SPILLED): the
 * complete lists, from the spill area the context keeps of its most recent b200tfs_parse_* call (the two-phase
 * parse re-runs itself with a larger spill area when a record needs it; the single-launch decode has none and
 * reports such a record as B200TFS_E_NONCANONICAL - decode it with the two-phase calls).  `dims` receives
 * min(cap, rank) entries; `runs` min(cap, n_runs) entries of the output's value field.  Outputs without the flag
 * are answered from the struct itself.                                                                        */
int b200tfs_output_dims(b200tfs_ctx* ctx, const b200tfs_output* out, int64_t* dims, int32_t cap);
int b200tfs_output_runs(b200tfs_ctx* ctx, const b200tfs_output* out, b200tfs_run* runs, int32_t cap);
/* Same walk for n bare TensorProto messages (tensor_proto_to_ndarray on a single message): one
 * output per record, key_len = 0.                                                                  */
int b200tfs_parse_tensor_protos(b200tfs_ctx* ctx, const void* arena_dev, int32_t n,
                                const uint64_t* rec_off, const uint64_t* rec_len, b200tfs_output* outs,
                                int32_t* rec_status);
/* Unpack m tabulated outputs into device buffers: out_rec_off[j] is the arena offset of the record
 * outs[j] came from (NULL: all zero); dst[j] receives outs[j].dst_bytes bytes (or
 * n_elems * sizeof(dst_dtype[j]) when dst_dtype[j] != outs[j].dtype and the cast is supported:
 * FLOAT -> HALF / BFLOAT16 round-to-nearest-even; NaNs as b200tfs_set_decode_cast describes).  status[j] (host, filled after an internal sync
 * only if `status` is non-NULL) reports per-output errors found while unpacking (element count
 * mismatch, integer out of range).  Async when status is NULL.                                    */
int b200tfs_unpack_outputs(b200tfs_ctx* ctx, const void* arena_dev, int32_t m, const b200tfs_output* outs,
                           const uint64_t* out_rec_off, void* const* dst_dev, const int32_t* dst_dtype,
                           int32_t* status);

/* Single-launch decode for the steady-state path: one kernel walks the tags AND moves the values,
 * with no host round trip.  Record i's fixed-width outputs (float_val / double_val / complex) are
 * written to dst_dev + i*dst_stride, each output 256-byte aligned in table order (b200tfs_output.dst_off);
 * outputs with varint or string values are tabulated only - finish those with b200tfs_unpack_outputs.
 * At most B200TFS_FUSED_MAX_OUTPUTS outputs per record.  Asynchronous and CUDA-graph capturable;
 * collect the table afterwards with b200tfs_decode_results (which synchronises).
 * Each launch remembers the framing of its record 0; records of the next launch that carry the same
 * framing skip the tag walk.  One corner is reported rather than decoded: a record that has exactly
 * that record's LENGTH but other framing, and whose values are spread over more 32 KB..256 KB tiles
 * than that record's, gets B200TFS_E_NONCANONICAL; decode it with the next launch (which starts
 * without a remembered framing) or with b200tfs_parse_responses + b200tfs_unpack_outputs.          */
#define B200TFS_FUSED_MAX_OUTPUTS 8
int b200tfs_decode_responses(b200tfs_ctx* ctx, const void* arena_dev, int32_t n, const uint64_t* rec_off,
                             const uint64_t* rec_len, void* dst_dev, uint64_t dst_stride);
/* Narrow on the way out (what a caller of the reference writes as tensor_proto_to_ndarray(...).astype(np.float16), tensors.py:42-46
 * followed by a host-side cast): after b200tfs_set_decode_cast(ctx, DT_HALF or DT_BFLOAT16) every DT_FLOAT output of
 * b200tfs_decode_responses / b200tfs_decode_responses_host_async on this context is written as fp16 / bf16 (IEEE round to nearest
 * even, the rounding of numpy's astype; b200tfs_output.dst_bytes = 2 * n_elems, .dtype stays DT_FLOAT, the wire's).  A NaN is
 * quieted first, as the reference's decode does, then becomes sign | 0x7E00 | ((w >> 13) & 0x3FF) in fp16 (numpy's astype) and
 * sign | 0x7FC0 in bf16 (ml_dtypes' astype).  Outputs of
 * other dtypes are unaffected.  DT_FLOAT (or 0) switches it off.  This is the decode half of BASELINE config C4 (a fp16 / bf16
 * tensor travels as DT_FLOAT); the encode half is b200tfs_tensor.src_dtype != wire_dtype.  No host involvement between the
 * launches and graph-capturable, like the uncast decode (the two-phase route - b200tfs_parse_responses +
 * b200tfs_unpack_outputs with dst_dtype - needs the host between its phases).  A batch of >= 4 MiB whose record length the
 * context has seen before runs as three launches (verify, guarded move, fallback: b200tfs_kernel_launches counts them); the
 * results and the table are the same.                                                               */
int b200tfs_set_decode_cast(b200tfs_ctx* ctx, int32_t float_as);
/* How the records of every b200tfs_decode_responses launch of this context were served so far (cumulative; synchronises):
 * by the framing template handed over in the kernel parameters (the host walked record 0 of a host-resident wire itself,
 * or adopted the previous launch's template from pinned memory while the stream was idle), by the template the previous
 * launch left in device memory, or by walking the tags.  Any pointer may be NULL.                                      */
int b200tfs_decode_stats(b200tfs_ctx* ctx, uint64_t* param_template, uint64_t* device_template, uint64_t* walked);
/* outs has n*B200TFS_FUSED_MAX_OUTPUTS slots; any pointer may be NULL.                             */
int b200tfs_decode_results(b200tfs_ctx* ctx, int32_t n, b200tfs_output* outs, int32_t* n_outs,
                           b200tfs_model_spec* specs, int32_t* rec_status);

/* ---- CUDA graphs: record a fixed sequence of encode / decode calls once, replay it per request ---
 * Between capture_begin and capture_end the asynchronous entry points (b200tfs_encode_requests,
 * b200tfs_encode_tensor_protos, b200tfs_decode_responses, b200tfs_memcpy_*) only record work; calls
 * that must synchronise (b200tfs_measure, the parse / *_host entry points, b200tfs_sync) fail with
 * B200TFS_E_ARG.  Run the same calls once before capturing so every scratch buffer has its final
 * size.  Plan images of batches too large for the kernel parameters get buffers of their own that
 * live until the context is destroyed.                                                             */
int b200tfs_capture_begin(b200tfs_ctx* ctx);
int b200tfs_capture_end(b200tfs_ctx* ctx, void** graph_exec);
int b200tfs_graph_launch(b200tfs_ctx* ctx, void* graph_exec);
int b200tfs_graph_destroy(void* graph_exec);
/* make every later call on ctx wait for an event recorded on another context's stream            */
int b200tfs_wait_event(b200tfs_ctx* ctx, void* ev);

/* ---- host-buffer convenience (what a client binds; H2D / D2H happen inside) -------------------- */
/* tensors[].data are HOST pointers (pinned or pageable).  Encodes n requests and leaves the wire
 * bytes in wire_host (capacity wire_cap); rec_off/rec_len as above.  Synchronous.                  */
int b200tfs_encode_requests_host(b200tfs_ctx* ctx, int32_t n, const b200tfs_request* reqs,
                                 void* wire_host, uint64_t wire_cap, uint64_t* rec_off,
                                 uint64_t* rec_len);
/* Same, but returns as soon as the copies and kernels are queued (it only blocks for the measure pass
 * when a packed-varint input of more than 4096 elements is present; smaller ones - labels, ids, a sequence
 * of token ids - are measured by the host, whose memory they are in): call b200tfs_sync before reading wire_host, which must be pinned
 * (b200tfs_host_alloc).  Two contexts running the _async entry points overlap H2D with D2H.
 *
 * Pipelining inside ONE call: a batch whose fixed-width payloads add up to at least 1 MiB (environment
 * B200TFS_PIPELINE_MIN, bytes; 0 = never) is cut into up to 8 slices of consecutive wire bytes; the
 * source bytes of slice k+1 travel host-to-device on a second stream while slice k is encoded and the
 * wire bytes of slice k-1 travel device-to-host on a third, so a single large request keeps both PCIe
 * directions busy.  The context's stream ends behind the last copy: b200tfs_sync (or an event recorded
 * on the context) covers everything, as before.  b200tfs_decode_responses_host_async does the same
 * for ONE response whose values lie in one fixed-width field.                                      */
int b200tfs_encode_requests_host_async(b200tfs_ctx* ctx, int32_t n, const b200tfs_request* reqs,
                                       void* wire_host, uint64_t wire_cap, uint64_t* rec_off,
                                       uint64_t* rec_len);
/* Host-buffer form of b200tfs_decode_responses: copies the n responses to the device, runs the fused
 * decode kernel and copies n*dst_stride bytes of decoded values back into dst_host (pinned), all
 * queued asynchronously.  b200tfs_decode_results then synchronises and returns the table.          */
int b200tfs_decode_responses_host_async(b200tfs_ctx* ctx, const void* wire_host, int32_t n,
                                        const uint64_t* rec_off, const uint64_t* rec_len,
                                        void* dst_host, uint64_t dst_stride);
/* how many *_host_async calls of this context took the sliced, three-stream path so far            */
int b200tfs_pipelined_calls(b200tfs_ctx* ctx, uint64_t* count);
/* Output straight into the caller's buffer: when wire_host (encode) / dst_host (decode) is page-locked memory the device can
 * address (b200tfs_host_alloc, cudaHostAlloc, cudaHostRegister), is 256-byte aligned and - encode - has room for the arena
 * layout (b200tfs_request_arena_size bytes: records start 256-byte aligned, so record 0 need not start at offset 0; read
 * rec_off), the kernels write it themselves with posted PCIe writes and no device-to-host copy is queued at all.  Pageable or unaligned buffers take the staged route as before.  B200TFS_DIRECT_OUT=0 or
 * b200tfs_set_pipeline(ctx, 0, 0) switches it off; this counts the calls that took it.                                                            */
int b200tfs_direct_calls(b200tfs_ctx* ctx, uint64_t* count);
/* Tune it per context: calls moving fewer than min_bytes of fixed-width payload stay monolithic (0 = never slice), at most
 * max_slices slices (2..8; default 4 - every slice costs about seven driver calls of host time).  A caller that keeps
 * several contexts busy at once already overlaps the two copy directions ACROSS calls and should switch slicing off: there the
 * slices only add driver calls, while a lone call gains from overlapping its own copies with its kernels.                    */
int b200tfs_set_pipeline(b200tfs_ctx* ctx, uint64_t min_bytes, int32_t max_slices);
int b200tfs_encode_tensor_protos_host(b200tfs_ctx* ctx, int32_t n, const b200tfs_tensor* tensors,
                                      void* wire_host, uint64_t wire_cap, uint64_t* rec_off,
                                      uint64_t* rec_len);
/* Decode n responses held in HOST memory: copies them to the device, parses, and returns the table
 * (offsets are relative to wire_host).  Follow with b200tfs_unpack_outputs_host.                   */
int b200tfs_parse_responses_host(b200tfs_ctx* ctx, const void* wire_host, int32_t n,
                                 const uint64_t* rec_off, const uint64_t* rec_len, int32_t max_outputs,
                                 b200tfs_output* outs, int32_t* n_outs, b200tfs_model_spec* specs,
                                 int32_t* rec_status);
int b200tfs_parse_tensor_protos_host(b200tfs_ctx* ctx, const void* wire_host, int32_t n,
                                     const uint64_t* rec_off, const uint64_t* rec_len,
                                     b200tfs_output* outs, int32_t* rec_status);
/* Unpack outputs of the most recent *_parse_*_host call on this context into HOST buffers.         */
int b200tfs_unpack_outputs_host(b200tfs_ctx* ctx, int32_t m, const b200tfs_output* outs,
                                const uint64_t* out_rec_off, void* const* dst_host,
                                const int32_t* dst_dtype, int32_t* status);

#ifdef __cplusplus
}
#endif
#endif /* B200TFS_H_ */
