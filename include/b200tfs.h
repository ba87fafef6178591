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
#define B200TFS_F_BROADCAST 0x10u     /* b200tfs_feature.flags: a 0-d column, whose one row is repeated in every example.
                                         b200tfs_tensor.flags (b200tfs_encode_padded_requests_async): the same tensor in every request */

/* ---- decode flags (b200tfs_output.flags, set by the parser) ----------------------------------- */
#define B200TFS_OF_TENSOR_CONTENT 0x1u /* values arrived in tensor_content                                        */
#define B200TFS_OF_MULTI_CHUNK 0x2u    /* values field split over several occurrences / unpacked elements         */
#define B200TFS_OF_UNPACKED 0x80u      /* some values arrived as unpacked scalar elements (wire type 0 / 1 / 5)   */
#define B200TFS_OF_SPILLED 0x100u      /* more dims than B200TFS_MAX_RANK and / or more value runs than B200TFS_MAX_RUNS: the rest
                                          is held by the context (b200tfs_output_dims / b200tfs_output_runs)               */
#define B200TFS_OF_DEVICE_VARINT 0x200u /* set by b200tfs_decode_results (b200tfs_set_decode_varints): the single-launch decode
                                           decoded this packed-varint output into its range itself; `status` is that decode's */
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

/* What a request's model_spec and PredictRequest.output_filter carry beside the name and version, for the _spec entry points
 * below (one per request, parallel to their reqs[]; NULL: none, the bytes of the entry point without _spec).  Strings are
 * written as given (UTF-8 by the caller), in field-number order: 0A name | 12 {08 version} | 1A signature_name | 22 version_label.
 *   signature_len  > 0: ModelSpec.signature_name (field 3); 0: not written (a proto3 scalar: empty is the default)
 *   version_label_len >= 0: ModelSpec.version_label (field 4, a version_choice oneof member: written even when empty, 22 00);
 *                     < 0: not set.  A label on a request with has_version is B200TFS_E_ARG.
 *   output_filter: n_output_filter names, written behind the last inputs entry as {1A vi(len) name}* in the given order (no
 *                  sorting, no de-duplication; an empty name is 1A 00).
 * A negative length, a NULL pointer behind a positive length or count: B200TFS_E_ARG.                                          */
typedef struct b200tfs_request_spec {
  const char* signature_name;
  int64_t signature_len;
  const char* version_label;
  int64_t version_label_len;
  const char* const* output_filter;
  const int64_t* output_filter_len;
  int64_t n_output_filter;
} b200tfs_request_spec;

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
  uint64_t n_strings;   /* string_val occurrences (unpacked on the host, or by b200tfs_decode_concat_strings) */
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
/* The same three with a b200tfs_request_spec per request (spec / specs: NULL = none; the forms above are these with NULL) */
int b200tfs_request_size_spec(const b200tfs_request* r, const b200tfs_request_spec* spec, uint64_t* total_len);
int b200tfs_request_frame_spec(const b200tfs_request* r, const b200tfs_request_spec* spec, void* buf, uint64_t cap, uint64_t* frame_len,
                               uint64_t* payload_off, uint64_t* payload_len, int32_t* perm);
int b200tfs_request_arena_size_spec(int32_t n, const b200tfs_request* reqs, const b200tfs_request_spec* specs, uint64_t* bytes);

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
 * kernels alone - count -> frame_requests_kernel (one thread per request runs the framing writers twice: once to count the
 * record and place it, once to write the framing and patch the destinations of the payload movers) -> move + emit - so the
 * call never synchronises and can be
 * captured in a CUDA graph (b200tfs_measure cannot).  Every record gets a 256-byte aligned slot sized for its worst case
 * (b200tfs_request_arena_size does that when it sees an unmeasured input) and lies inside it with its largest payload
 * 128-byte aligned; WHERE exactly, and how long it is, is known once the kernels have run: b200tfs_encode_results
 * synchronises and delivers rec_off / rec_len (or the first per-request error).  Bytes identical to b200tfs_encode_requests. */
int b200tfs_encode_requests_async(b200tfs_ctx* ctx, int32_t n, const b200tfs_request* reqs, void* arena_dev,
                                  uint64_t arena_cap);
int b200tfs_encode_results(b200tfs_ctx* ctx, int32_t n, uint64_t* rec_off, uint64_t* rec_len);
/* What frame_requests_kernel computes for ONE request, run on the host (the same inline function; needs no device): given the
 * packed length of every packed-varint input (packed_len[i] for inputs[i]; other entries ignored) it writes every framing
 * byte of the record into buf at the place it has on the wire and reports where the record lies (rec_off / rec_len) and,
 * per input, where the framing writers put its payload (payload_off[i] / payload_len[i]; 0 / 0 for an input without values). */
int b200tfs_request_frame_deferred(const b200tfs_request* r, const uint64_t* packed_len, void* buf, uint64_t cap,
                                   uint64_t* rec_off, uint64_t* rec_len, uint64_t* payload_off, uint64_t* payload_len);
/* The same two with a b200tfs_request_spec per request (NULL: none).  The output_filter run lies behind the last payload, so
 * where it goes depends on the lengths the device counts: frame_requests_kernel copies it there from the host-built bytes. */
int b200tfs_encode_requests_async_spec(b200tfs_ctx* ctx, int32_t n, const b200tfs_request* reqs, const b200tfs_request_spec* specs,
                                       void* arena_dev, uint64_t arena_cap);
int b200tfs_request_frame_deferred_spec(const b200tfs_request* r, const b200tfs_request_spec* spec, const uint64_t* packed_len, void* buf,
                                        uint64_t cap, uint64_t* rec_off, uint64_t* rec_len, uint64_t* payload_off, uint64_t* payload_len);

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
 * outputs with varint or string values are tabulated only - finish those with b200tfs_unpack_outputs (or, for the
 * varint ones, switch on b200tfs_set_decode_varints).
 * At most B200TFS_FUSED_MAX_OUTPUTS outputs per record.  Asynchronous and CUDA-graph capturable;
 * collect the table afterwards with b200tfs_decode_results (which synchronises).
 * Each launch remembers the framing of its record 0; records of the next launch that carry the same
 * framing skip the tag walk.  One corner is reported rather than decoded: a record that has exactly
 * that record's LENGTH but other framing, and whose values are spread over more tiles (32 KB or 64 KB
 * each, or B200TFS_TILE_BYTES) than that record's, gets B200TFS_E_NONCANONICAL; decode it with the next launch (which starts
 * without a remembered framing) or with b200tfs_parse_responses + b200tfs_unpack_outputs.
 * The launch stores only into [dst_off, dst_off + dst_bytes) of the B200TFS_OK fixed-width outputs of B200TFS_OK records:
 * every other byte of every slot - all of it for a record that did not decode - keeps what the caller left there.
 * With b200tfs_set_decode_varints(ctx, 1) the packed-varint outputs get ranges of their own as well (see there); a
 * varint output stores only inside its own range, and when its status is not B200TFS_OK that range's contents are
 * unspecified.                                                                                                       */
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
/* Decode packed-varint outputs too (int_val, int64_val, uint32_val, uint64_val, bool_val, half_val): after
 * b200tfs_set_decode_varints(ctx, 1) every later b200tfs_decode_responses / b200tfs_decode_responses_host_async of this
 * context also decodes them, still without the host between its launches and still graph-capturable (0 switches it off;
 * allowed before a capture, not during one).  Layout: every B200TFS_OK varint output with n_elems > 0 gets a 256-byte aligned
 * range [dst_off, dst_off + dst_bytes) of the record's slot, in table order together with the fixed-width outputs
 * (dst_bytes = n_elems * element size in memory; a range that does not fit dst_stride: B200TFS_E_SIZE).  Values: what
 * b200tfs_unpack_outputs writes with dst_dtype NULL (int_val truncated to int32, bool normalised, half_val as TF bit
 * patterns).  b200tfs_decode_results then reports, for every output decoded this way, B200TFS_OF_DEVICE_VARINT in `flags`
 * and in `status`: B200TFS_OK; B200TFS_E_SHAPE (value count != n_elems); B200TFS_E_PARSE (a malformed varint; wins over
 * E_SHAPE); B200TFS_E_RANGE (a value that does not fit the dtype); B200TFS_E_NONCANONICAL (values in rows of unpacked
 * elements: finish that output with b200tfs_unpack_outputs).  The launch appends three kernels (plan, count, emit - the
 * two-phase route's own decoders over tables built on the device) and one status copy; b200tfs_kernel_launches counts them.
 * b200tfs_decode_results folds those statuses in when the most recent b200tfs_decode_responses* CALL on the context ran with the
 * switch on - like the record count it answers for, that is the last call, not the last graph replayed: replay a graph captured
 * with the switch on after an eager call with it off, and its varint outputs read as tabulated only (their ranges are written). */
int b200tfs_set_decode_varints(b200tfs_ctx* ctx, int32_t on);
/* What dst_stride the single-launch decode needs for n records in HOST memory (needs no device): the records are walked and laid out
 * as the launch lays them out (varints != 0: with b200tfs_set_decode_varints on), with no cast; *slot_bytes receives the most bytes
 * any record's slot uses (round up to 256 for dst_stride), *n_varint_outputs (may be NULL) how many varint ranges the batch has -
 * 0: the switch would decode nothing more.  Records that do not walk (malformed, more than B200TFS_FUSED_MAX_OUTPUTS outputs)
 * count 0 bytes: the launch does not decode them either.                                                                   */
int b200tfs_decode_slot_bytes(const void* wire_host, int32_t n, const uint64_t* rec_off, const uint64_t* rec_len, int32_t varints,
                              uint64_t* slot_bytes, int32_t* n_varint_outputs);
/* How the records of every b200tfs_decode_responses launch of this context were served so far (cumulative; synchronises):
 * by the framing template handed over in the kernel parameters (the host walked record 0 of a host-resident wire itself,
 * or adopted the previous launch's template from pinned memory while the stream was idle), by the template the previous
 * launch left in device memory, or by walking the tags.  Any pointer may be NULL.                                      */
int b200tfs_decode_stats(b200tfs_ctx* ctx, uint64_t* param_template, uint64_t* device_template, uint64_t* walked);
/* outs has n*B200TFS_FUSED_MAX_OUTPUTS slots; any pointer may be NULL.                             */
int b200tfs_decode_results(b200tfs_ctx* ctx, int32_t n, b200tfs_output* outs, int32_t* n_outs,
                           b200tfs_model_spec* specs, int32_t* rec_status);

/* ---- batch decode into one tensor per output, concatenated along axis 0 ---------------------------
 * What a client that split a batch into n requests wants back: for each requested key, the outputs of every record
 * concatenated along their first dimension - np.concatenate([decode(w)[key] for w in wires], axis=0) - written straight into
 * one device buffer per key, every payload byte read once and written once.  Record r's rows start where the rows of
 * records 0..r-1 end; since those counts are only known once the records are parsed, the destinations are planned on the
 * device (a replayed CUDA graph adapts to new row counts).  Only the requested outputs are decoded.                       */
#define B200TFS_CONCAT_MAX_KEYS 8
typedef struct b200tfs_concat_key {
  const char* key;        /* in: map key bytes (not NUL terminated); the keys of one call must be distinct            */
  int64_t key_len;
  void* dst;              /* in: b200tfs_decode_concat*: device destination of the concatenated tensor               */
  uint64_t dst_cap;       /* in: its capacity in bytes - nothing is ever stored at or past dst + dst_cap              */
  int32_t dtype;          /* out (b200tfs_concat_layout): DT_* of the first record that has the key                   */
  int32_t rank;           /* out: rank of the concatenated tensor                                                     */
  int64_t dims[B200TFS_MAX_RANK]; /* out: dims[0] = rows of all records together, the rest those of every record      */
  uint64_t bytes;         /* out: bytes of the concatenated tensor in memory (2 per float32 element with a cast)      */
  int32_t status;         /* out: B200TFS_OK (also for a DT_STRING key: bytes 0, decoded on the host - or, with
                             b200tfs_concat_strings entries, bytes of its int64 offsets) or the first
                             problem in record order: the record's error (E_PARSE, ...,
                             E_NONCANONICAL for a record the device route cannot tabulate: more than
                             B200TFS_FUSED_MAX_OUTPUTS outputs, rank > B200TFS_MAX_RANK, more than B200TFS_MAX_RUNS runs),
                             the output's tabulated error (E_SHAPE, E_KEY, ...), E_KEY when the record lacks the key,
                             E_SHAPE for rank 0 / another rank / other trailing dims, E_DTYPE for another dtype            */
  int32_t bad_rec;        /* out: the record `status` is about (-1 when OK)                                          */
} b200tfs_concat_key;
/* Host only (needs no device): walks the n records in host memory and fills the out fields of keys[0..n_keys), which is what
 * a caller needs to allocate exact-size destinations.  cast: 0, or DT_HALF / DT_BFLOAT16 as b200tfs_set_decode_cast sets it. */
int b200tfs_concat_layout(const void* wire_host, int32_t n, const uint64_t* rec_off, const uint64_t* rec_len, int32_t n_keys,
                          b200tfs_concat_key* keys, int32_t cast);
/* The keys of one record in host memory, in table order (the order of their first map entry): key_off[i] (from the start of
 * the record) and key_len[i] for i < *count; at most `cap` are written.  A record that does not walk: its error.            */
int b200tfs_response_keys(const void* rec_host, uint64_t rec_len, int32_t cap, uint64_t* key_off, uint32_t* key_len,
                          int32_t* count);
/* Decode n PredictResponses of the device arena into keys[k].dst for every k < n_keys (<= B200TFS_CONCAT_MAX_KEYS; only the
 * in fields are read).  Asynchronous and CUDA-graph capturable: the host is not involved between the launches (parse,
 * one-CTA plan, move engine, packed-varint plan / count / emit - b200tfs_kernel_launches counts six).  The scratch it needs
 * is sized from n, n_keys and rec_len alone, so a graph captured once serves any records of those lengths.  Float32 outputs
 * are narrowed per b200tfs_set_decode_cast.  Values: what b200tfs_unpack_outputs writes with dst_dtype NULL (half_val as TF
 * bit patterns).  Stores: only into [dst_off, dst_off + dst_bytes) of the (record, key) pairs b200tfs_concat_results reports
 * B200TFS_OK, or reports with B200TFS_OF_DEVICE_VARINT (a packed-varint output whose place was reserved; when its decode
 * failed the contents are unspecified), never at or past dst_cap.  Every other byte keeps what the caller left there.      */
int b200tfs_decode_concat(b200tfs_ctx* ctx, const void* arena_dev, int32_t n, const uint64_t* rec_off, const uint64_t* rec_len,
                          int32_t n_keys, const b200tfs_concat_key* keys);
/* The same for records in host memory: the wire is copied to the device inside (asynchronous; wire_host should be pinned). */
int b200tfs_decode_concat_host_async(b200tfs_ctx* ctx, const void* wire_host, int32_t n, const uint64_t* rec_off,
                                     const uint64_t* rec_len, int32_t n_keys, const b200tfs_concat_key* keys);
/* Results of the context's most recent b200tfs_decode_concat* call (synchronises).  outs[r * n_keys + k]: record r's table entry
 * for key k, with dst_off = where its rows start inside keys[k].dst and `status`: B200TFS_OK (decoded); the record's or the
 * output's error; B200TFS_E_KEY (no such key); B200TFS_E_DTYPE / B200TFS_E_SHAPE (dtype / rank / trailing dims differ from the
 * first record that decoded the key; rank 0); B200TFS_E_SIZE (its rows end past dst_cap); B200TFS_E_NONCANONICAL, which is
 * either a packed-varint output in rows of unpacked elements (its place [dst_off, dst_off + dst_bytes) is reserved; finish it
 * with b200tfs_unpack_outputs there), a string output of a call without b200tfs_concat_strings entries (nothing reserved: such
 * strings are decoded on the host; see b200tfs_decode_concat_strings for the string pairs of a call with them), or a record the
 * device parse cannot tabulate (more than B200TFS_FUSED_MAX_OUTPUTS outputs, rank > B200TFS_MAX_RANK, more than
 * B200TFS_MAX_RUNS runs; nothing reserved).  Outputs the tolerant decode would accept although their table entry is an error -
 * tensor_content only, fewer fixed-width values than the shape holds (TF's padding) - keep that error (B200TFS_E_SHAPE) and
 * get no place: whether to accept them is the caller's policy, and the row count of such a batch is only known once it is
 * chosen.  Packed-varint outputs carry B200TFS_OF_DEVICE_VARINT and that decode's status.  specs[r] and rec_status[r] as
 * b200tfs_parse_responses gives them; any pointer may be NULL.                                                           */
int b200tfs_concat_results(b200tfs_ctx* ctx, int32_t n, int32_t n_keys, b200tfs_output* outs, b200tfs_model_spec* specs,
                           int32_t* rec_status);

/* DT_STRING outputs of the same decode, as offset-indexed byte columns (the Arrow / cuDF layout b200tfs_bytes reads): for a key
 * whose outputs are DT_STRING, the string_val elements of every record, in record order, as raw bytes (no UTF-8 check; NULs and
 * high bytes kept).  With m strings of D bytes in all, keys[k].dst receives int64 offsets[m + 1] (offsets[0] = 0, string j is
 * data[offsets[j], offsets[j + 1])) and the entry's `data` the D bytes.  The offsets take the key's own dst / dst_cap so that
 * b200tfs_output.dst_off keeps its meaning: the byte offset of the record's first offset entry (8 * its first string).  One entry
 * per key, parallel to keys; entries of keys whose outputs are not DT_STRING are ignored.                                         */
typedef struct b200tfs_concat_strings {
  void* data;             /* in: device destination of the key's string bytes                                                  */
  uint64_t data_cap;      /* in: its capacity in bytes - nothing is ever stored at or past data + data_cap                     */
  uint64_t strings;       /* out (b200tfs_concat_strings_layout): m, the strings of every record together                     */
  uint64_t data_bytes;    /* out: D, their bytes                                                                               */
} b200tfs_concat_strings;
/* b200tfs_concat_layout with entries (strings == NULL: that call itself).  A DT_STRING key that lays out gets `strings` and
 * `data_bytes`, and keys[k].bytes = 8 * (strings + 1), the offsets' size.  A record whose string_val elements the device walk
 * does not find in its last `value` occurrence (a map entry that carries its TensorProto in several, which the runtime merges)
 * is B200TFS_E_NONCANONICAL: that batch is decoded on the host.                                                                  */
int b200tfs_concat_strings_layout(const void* wire_host, int32_t n, const uint64_t* rec_off, const uint64_t* rec_len, int32_t n_keys,
                                  b200tfs_concat_key* keys, b200tfs_concat_strings* strings, int32_t cast);
/* Host only, closed form from the record lengths alone, for a caller that captures a graph once: every string_val element takes at
 * least two bytes of wire and its bytes lie in the wire, so one key of any records of these lengths has at most *max_strings
 * strings (offsets of 8 * (*max_strings + 1) bytes) and *max_data_bytes bytes.  Either pointer may be NULL.                    */
int b200tfs_concat_strings_bound(int32_t n, const uint64_t* rec_len, uint64_t* max_strings, uint64_t* max_data_bytes);
/* b200tfs_decode_concat with entries (strings == NULL: that call itself).  Still asynchronous and CUDA-graph capturable with no
 * host step between the launches: the plan places every (record, string key)'s offsets, then four kernels (index: a warp per
 * pair walks its string_val elements; scan: one CTA places their bytes; copy; fix: the final offsets) follow the plan and come
 * ahead of the varint tail - b200tfs_kernel_launches counts ten.  The scratch is sized from n, n_keys and rec_len alone, so a
 * replay over new records of the same lengths re-plans string counts and byte offsets.  b200tfs_concat_results reports each
 * (record, string key): B200TFS_OK with dst_off = 8 * its first string and dst_bytes = 8 * its strings; B200TFS_E_SIZE when its
 * offsets (up to and including the entry behind its last string) would end past dst_cap or its bytes past data_cap (a pair's bytes
 * hold their place whether or not they fit, so every later pair of the key that decoded, one of no bytes too, starts past
 * data_cap and is B200TFS_E_SIZE as well); or
 * B200TFS_E_NONCANONICAL when its string_val elements do not all lie in its last `value` occurrence (decode that batch on the
 * host).  Stores: for the OK pairs, their offset entries and bytes, and offsets[m] behind the last OK pair of the key; the entries
 * of a pair that ends B200TFS_E_SIZE for its bytes or B200TFS_E_NONCANONICAL may hold scratch values.  Nothing at or past dst_cap
 * or data_cap.                                                                                                                     */
int b200tfs_decode_concat_strings(b200tfs_ctx* ctx, const void* arena_dev, int32_t n, const uint64_t* rec_off, const uint64_t* rec_len,
                                  int32_t n_keys, const b200tfs_concat_key* keys, const b200tfs_concat_strings* strings);
int b200tfs_decode_concat_strings_host_async(b200tfs_ctx* ctx, const void* wire_host, int32_t n, const uint64_t* rec_off,
                                             const uint64_t* rec_len, int32_t n_keys, const b200tfs_concat_key* keys,
                                             const b200tfs_concat_strings* strings);

/* ---- batch decode into one padded tensor per output (ragged trailing dims) --------------------------
 * What a caller of a sequence model wants back (per-token logits f32[1, T_r, V], token ids int64[1, T_r], ...): for each requested
 * key, the outputs of every record concatenated along axis 0 with every other axis padded - record r's output lands in rows
 * [first_row, first_row + dims[0]) of one tensor of shape [rows, dims[1], ..., dims[rank-1]], at index 0 of every trailing axis, and
 * every other element of those rows holds the pad element.  As for the concatenated decode, the rows and the trailing dims are
 * planned on the device, so a replayed CUDA graph adapts to new records.  Only the requested outputs are decoded.              */
typedef struct b200tfs_pad_key {
  const char* key;        /* in: map key bytes (not NUL terminated); the keys of one call must be distinct                   */
  int64_t key_len;
  void* dst;              /* in: b200tfs_decode_padded*: device destination, 16-byte aligned                                  */
  uint64_t dst_cap;       /* in: its capacity in bytes - nothing is ever stored at or past dst + dst_cap                      */
  int32_t dtype;          /* out (b200tfs_padded_layout): DT_* of the first record that has the key                          */
  int32_t rank;           /* out: its rank.  In (b200tfs_decode_padded*): the destination's rank                              */
  int64_t dims[B200TFS_MAX_RANK]; /* out: dims[0] = rows of all records together, dims[1..rank) the elementwise maximum of the
                             records' trailing dims.  In (b200tfs_decode_padded*): dims[1..rank) are the destination's trailing
                             dims (a caller that captures a graph fixes them once, e.g. at the model's longest sequence)     */
  uint64_t bytes;         /* out: rows * prod(dims[1..rank)) * element size in memory (2 for float32 with a cast)              */
  int32_t status;         /* out: as b200tfs_concat_key.status, except that other trailing dims are not an error (a DT_STRING
                             key: OK with bytes 0, decoded on the host - or, with b200tfs_padded_strings entries, bytes of
                             its int64 offsets)                                                                              */
  int32_t bad_rec;        /* out: the record `status` is about (-1 when OK)                                                  */
  uint8_t pad_bits[16];   /* in: the pad element's bit pattern in the destination dtype (little-endian; the first element
                             size bytes are used)                                                                            */
} b200tfs_pad_key;
/* Host only (needs no device): walks the n records in host memory and fills the out fields of keys[0..n_keys).  The first
 * problem in record order, with b200tfs_concat_layout's codes: E_SHAPE (rank 0, another rank), E_DTYPE, E_KEY, the output's
 * tabulated error, E_NONCANONICAL (a record the device route cannot tabulate).  cast: 0, or DT_HALF / DT_BFLOAT16.              */
int b200tfs_padded_layout(const void* wire_host, int32_t n, const uint64_t* rec_off, const uint64_t* rec_len, int32_t n_keys,
                          b200tfs_pad_key* keys, int32_t cast);
/* Decode n PredictResponses of the device arena into keys[k].dst for every k < n_keys (<= B200TFS_CONCAT_MAX_KEYS; only the in
 * fields are read).  Asynchronous and CUDA-graph capturable, with no host step between the launches (parse, one-CTA plan,
 * destination-major emit, packed-varint plan / count / emit - b200tfs_kernel_launches counts six).  The scratch is sized from n,
 * n_keys and rec_len alone, so a replay over new records of the same lengths re-plans rows and trailing dims.  Float32 outputs are
 * narrowed per b200tfs_set_decode_cast; values are what b200tfs_decode_concat writes.  Stores: with `pitch` = prod(dims[1..rank))
 * * element size and rows_used = the rows of the records that got a place, every byte of [0, rows_used * pitch) of keys[k].dst is
 * written exactly once - values and pads alike - and nothing else, never at or past dst_cap.  A record whose trailing dim exceeds
 * dims[d], or whose rows would pass dst_cap, is B200TFS_E_SIZE and gets no place.  A packed-varint output whose decode fails
 * leaves its value elements unspecified (its pads are written).                                                                  */
int b200tfs_decode_padded(b200tfs_ctx* ctx, const void* arena_dev, int32_t n, const uint64_t* rec_off, const uint64_t* rec_len,
                          int32_t n_keys, const b200tfs_pad_key* keys);
/* The same for records in host memory: the wire is copied to the device inside (asynchronous; wire_host should be pinned). */
int b200tfs_decode_padded_host_async(b200tfs_ctx* ctx, const void* wire_host, int32_t n, const uint64_t* rec_off,
                                     const uint64_t* rec_len, int32_t n_keys, const b200tfs_pad_key* keys);
/* Results of the context's most recent b200tfs_decode_padded* call (synchronises).  outs[r * n_keys + k]: record r's table entry
 * for key k - its `dims` are that record's own shape - with dst_off = the byte offset of its first row inside keys[k].dst,
 * dst_bytes = the bytes of its rows there, and `status` as b200tfs_concat_results words it, except that other trailing dims are not
 * an error and that packed-varint rows of unpacked elements are B200TFS_E_NONCANONICAL with no place.  specs[r] and rec_status[r]
 * as b200tfs_parse_responses gives them; any pointer may be NULL.                                                               */
int b200tfs_padded_results(b200tfs_ctx* ctx, int32_t n, int32_t n_keys, b200tfs_output* outs, b200tfs_model_spec* specs,
                           int32_t* rec_status);

/* DT_STRING outputs of the same decode, as one padded offset-indexed byte column per key (the b200tfs_bytes layout): for a key whose
 * outputs are DT_STRING, position (row, i_1, ..., i_{rank-1}) of the [rows, dims[1], ..., dims[rank-1]] destination holds, in C
 * order, record r's string at (row - first_row, i_1, ...) when every index lies inside its own dims, and the pad string otherwise
 * (raw bytes; no UTF-8 check).  With m = rows * prod(dims[1..rank)) positions, keys[k].dst receives int64 offsets[m + 1]
 * (offsets[0] = 0, position p is data[offsets[p], offsets[p + 1])) and the entry's `data` the bytes, so that
 * b200tfs_output.dst_off keeps its meaning: the byte offset of the record's first row, 8 bytes per position.  One entry per key,
 * parallel to keys; entries of keys whose outputs are not DT_STRING are ignored, and so are those keys' pad_bits.              */
typedef struct b200tfs_padded_strings {
  void* data;             /* in: device destination of the key's string bytes                                                  */
  uint64_t data_cap;      /* in: its capacity in bytes - nothing is ever stored at or past data + data_cap                     */
  const void* pad;        /* in: the pad string's bytes in host memory (copied inside the call; NULL when pad_len is 0)        */
  uint64_t pad_len;       /* in: its length                                                                                    */
  uint64_t strings;       /* out (b200tfs_padded_strings_layout): the records' own strings together                            */
  uint64_t data_bytes;    /* out: their bytes                                                                                  */
} b200tfs_padded_strings;
/* b200tfs_padded_layout with entries (strings == NULL: that call itself).  A DT_STRING key that lays out gets `strings` and
 * `data_bytes`, and keys[k].bytes = 8 * (m + 1), the offsets' size, with m = dims[0] * prod(dims[1..rank)) of the elementwise
 * maximum.  Its column then takes data_bytes + (m - strings) * pad_len data bytes; with other trailing dims D (pad_to), m is
 * dims[0] * prod(D).  A record whose string_val elements the device walk does not find in its last `value` occurrence is
 * B200TFS_E_NONCANONICAL, as for b200tfs_concat_strings_layout.  For a caller that captures a graph once with trailing dims D and
 * at most R rows: offsets of 8 * (R * prod(D) + 1) bytes and max_data_bytes + R * prod(D) * pad_len data bytes hold any records
 * of the same lengths (max_data_bytes from b200tfs_concat_strings_bound).                                                     */
int b200tfs_padded_strings_layout(const void* wire_host, int32_t n, const uint64_t* rec_off, const uint64_t* rec_len, int32_t n_keys,
                                  b200tfs_pad_key* keys, b200tfs_padded_strings* strings, int32_t cast);
/* b200tfs_decode_padded with entries (strings == NULL: that call itself).  Still asynchronous and CUDA-graph capturable with no host
 * step between the launches: the plan places every (record, string key)'s rows as for a numeric key, then four kernels (index: a
 * warp per pair walks its string_val elements and notes each at its padded position; scan: one CTA places every record's bytes,
 * its own and its pads'; copy: strings and pads, destination-major; fix: the final offsets of the own strings) come ahead of the
 * varint tail - b200tfs_kernel_launches counts ten.  The scratch is sized from n, n_keys and rec_len alone: a replay over new
 * records of the same lengths re-plans rows, string counts and bytes.  b200tfs_padded_results reports each (record, string key):
 * B200TFS_OK with dst_off / dst_bytes of its rows; B200TFS_E_SIZE when its rows would end past dst_cap (the entry behind them
 * included), its bytes past data_cap, or a trailing dim exceeds the destination's - it gets no place, and the rows in use end at
 * the first record that ends B200TFS_E_SIZE for its bytes; or B200TFS_E_NONCANONICAL when its string_val elements do not all lie
 * in its last `value` occurrence (its rows then hold the pad string: decode that batch on the host).  Stores: with rows_used the
 * rows in use, every offset entry of [0, rows_used * prod(dims[1..rank))] and every data byte of those rows, each once; the
 * entries of a record that ends B200TFS_E_SIZE for its bytes may hold scratch values.  Nothing at or past dst_cap or data_cap. */
int b200tfs_decode_padded_strings(b200tfs_ctx* ctx, const void* arena_dev, int32_t n, const uint64_t* rec_off, const uint64_t* rec_len,
                                  int32_t n_keys, const b200tfs_pad_key* keys, const b200tfs_padded_strings* strings);
int b200tfs_decode_padded_strings_host_async(b200tfs_ctx* ctx, const void* wire_host, int32_t n, const uint64_t* rec_off,
                                             const uint64_t* rec_len, int32_t n_keys, const b200tfs_pad_key* keys,
                                             const b200tfs_padded_strings* strings);

/* ---- batch encode of PredictRequests cut out of one padded tensor per input ------------------------
 * The inverse of b200tfs_decode_padded: request r's tensor for a padded input P of shape [R, D_1, ..., D_{m-1}] is the box
 * P[r0 : r0 + S[r,0], :S[r,1], ..., :S[r,m-1]], r0 = S[0,0] + ... + S[r-1,0], where S (int64[n, m] in device memory, or int64[n] row
 * counts with every trailing dim full) gives each request's shape.  The bytes are what b200tfs_encode_requests writes for the
 * request of those boxes.  Each input's b200tfs_tensor describes the padded tensor (device `data`, `dims` = [R, D_1, ...], dtypes,
 * flags, key); with B200TFS_F_BROADCAST (0x10, the b200tfs_feature flag) in its flags it is the same tensor, dims as given (any
 * rank, 0 included), in every request.  The shapes are only read on the device, so a replayed CUDA graph re-plans rows, boxes,
 * framing and record offsets from whatever the shapes tables and the tensors hold then.                                        */
typedef struct b200tfs_pad_input {
  const int64_t* shapes;  /* b200tfs_encode_padded_requests_async: device int64[n, cols]; b200tfs_padded_request_frame: host, the one
                             request's `cols` entries.  Ignored for a B200TFS_F_BROADCAST input                                         */
  int32_t cols;           /* the input's rank (full shapes) or 1 (row counts)                                                        */
  int32_t pad_;
} b200tfs_pad_input;
/* Host only, closed form from n and the padded shapes: arena bytes that always hold the n records (per padded input the whole
 * tensor's payload - 10 bytes per element for the packed-varint dtypes - since the boxes partition its rows; per request the
 * largest framing these dims allow plus 256 + 128 bytes of placement; broadcast payloads n times).                               */
int b200tfs_padded_request_arena_size(int32_t n, const b200tfs_request* req, uint64_t* bytes);
/* Encode the n requests into the device arena (256-byte aligned, arena_cap bytes).  `req` gives the model spec, order, flags and
 * inputs (at most B200TFS_CONCAT_MAX_KEYS padded and B200TFS_CONCAT_MAX_KEYS broadcast inputs, ranks 1..B200TFS_MAX_RANK - 0 too
 * for broadcast - no DT_STRING: B200TFS_E_ARG / B200TFS_E_DTYPE), in[i] the shapes of req->inputs[i].  Kernels only (plan, varint
 * count, layout, frame, move, varint emit; b200tfs_kernel_launches counts them): never synchronises and can be captured.  Records
 * are placed one behind the other in request order, each slot 256-byte aligned with the largest payload 128-byte aligned.
 * Collect rec_off / rec_len and the first per-request error with b200tfs_encode_results: B200TFS_E_SHAPE (a negative dim, a
 * trailing dim past the padded one), B200TFS_E_SIZE (rows past R: that request and every later one), B200TFS_E_TOOBIG (over
 * 2 GiB).  A request with an error gets rec_len 0 and no bytes; stores go only into [rec_off, rec_off + rec_len) of the others. */
int b200tfs_encode_padded_requests_async(b200tfs_ctx* ctx, int32_t n, const b200tfs_request* req, const b200tfs_pad_input* in,
                                         void* arena_dev, uint64_t arena_cap);
/* What the framing kernels do for ONE request, run on the host (the same inline code; needs no device): in[i].shapes points at the
 * request's host shape row for req->inputs[i], packed_len[i] stands in for the counted packed length of a packed-varint input.
 * Writes every framing byte of the record at its wire position in buf (the payload ranges are left alone), and reports the record
 * length and, per input, where its payload starts and how long it is.  The request's rows start at row 0 of each padded input.     */
int b200tfs_padded_request_frame(const b200tfs_request* req, const b200tfs_pad_input* in, const uint64_t* packed_len, void* buf,
                                 uint64_t cap, uint64_t* rec_len, uint64_t* payload_off, uint64_t* payload_len);
/* The same three with DT_STRING inputs from string columns (the b200tfs_bytes layout below; bytes == NULL: those calls
 * themselves).  bytes[i] goes with req->inputs[i]; offsets == NULL: not a string column.  A string input has src_dtype and
 * wire_dtype DT_STRING, `data` is its byte buffer (data_len bytes, device memory for the _async call), `offsets` device int64[m + 1]
 * for the m strings that fill `dims` in C order, and offsets[0] need not be 0 (a sliced column).  It is cut into boxes like any
 * padded input (or is the same tensor in every request with B200TFS_F_BROADCAST), and each string of a box becomes one string_val
 * value of its raw bytes, in C order (a box of no strings writes no string_val).
 * A request's box reads, in this order, the offset of its first row's start, both ends of every string of the box, and its last
 * row's end (a broadcast input: every offset), and they must satisfy
 *     0 <= each offset <= data_len, and no offset read is smaller than the one read before it,
 * so that the boxes of a call take disjoint byte ranges: the arena holds per padded string input data_len + 11 * strings bytes, per
 * broadcast one n * (data_len + 11 * strings).  The kernels check this, and clamp every offset into [0, data_len] first, so no read
 * leaves [data, data + data_len); a request that breaks it gets B200TFS_E_SHAPE in b200tfs_encode_results and no bytes (no store
 * leaves [rec_off, rec_off + rec_len) of the others).  Such a request can let its neighbours read overlapping bytes, so that the
 * good requests together need more than the arena bound: the later ones then get B200TFS_E_SIZE rather than their bytes.  Offsets that no box reads are never looked at.  A replayed CUDA graph
 * follows new shapes, data and offsets as long as data_len and the column's dims stay the same.  A call with a string input
 * launches two kernels more (string count and string emit).  In b200tfs_padded_request_frame_columns packed_len[i] stands in for
 * the counted bytes of a string input's values (sum of 1 + varint(len) + len), as for a packed-varint input, and the offsets are not
 * read.  A DT_STRING input without an entry: B200TFS_E_DTYPE; an entry on another dtype, a wire dtype other than DT_STRING,
 * B200TFS_F_TENSOR_CONTENT / B200TFS_F_KEEP_SNAN on a string input, offsets not 8-byte aligned, a negative data_len or bytes flags
 * other than B200TFS_F_DEVICE_DATA: B200TFS_E_ARG - all checked before the context's device is used.                            */
struct b200tfs_bytes;   /* defined with the tf.Example string columns, below */
int b200tfs_padded_request_columns_arena_size(int32_t n, const b200tfs_request* req, const struct b200tfs_bytes* bytes, uint64_t* out);
int b200tfs_encode_padded_requests_columns_async(b200tfs_ctx* ctx, int32_t n, const b200tfs_request* req, const b200tfs_pad_input* in,
                                                 const struct b200tfs_bytes* bytes, void* arena_dev, uint64_t arena_cap);
int b200tfs_padded_request_frame_columns(const b200tfs_request* req, const b200tfs_pad_input* in, const struct b200tfs_bytes* bytes,
                                         const uint64_t* packed_len, void* buf, uint64_t cap, uint64_t* rec_len,
                                         uint64_t* payload_off, uint64_t* payload_len);
/* The same three with one b200tfs_request_spec for every request of the call (NULL: none; the _columns forms are these with
 * NULL).  The output_filter run follows each record's last payload, so the framing kernels place it from the device shapes. */
int b200tfs_padded_request_columns_arena_size_spec(int32_t n, const b200tfs_request* req, const struct b200tfs_bytes* bytes,
                                                   const b200tfs_request_spec* spec, uint64_t* out);
int b200tfs_encode_padded_requests_columns_async_spec(b200tfs_ctx* ctx, int32_t n, const b200tfs_request* req, const b200tfs_pad_input* in,
                                                      const struct b200tfs_bytes* bytes, const b200tfs_request_spec* spec, void* arena_dev,
                                                      uint64_t arena_cap);
int b200tfs_padded_request_frame_columns_spec(const b200tfs_request* req, const b200tfs_pad_input* in, const struct b200tfs_bytes* bytes,
                                              const b200tfs_request_spec* spec, const uint64_t* packed_len, void* buf, uint64_t cap,
                                              uint64_t* rec_len, uint64_t* payload_off, uint64_t* payload_len);

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
/* b200tfs_encode_requests_host with a b200tfs_request_spec per request (NULL: none).  The output_filter run is the last framing
 * bytes of each record, written with the record's other framing (the first slice of a pipelined call).                     */
int b200tfs_encode_requests_host_spec(b200tfs_ctx* ctx, int32_t n, const b200tfs_request* reqs, const b200tfs_request_spec* specs,
                                      void* wire_host, uint64_t wire_cap, uint64_t* rec_off, uint64_t* rec_len);
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

/* ---- Classify / Regress requests: a batch of tf.Examples from columnar arrays -----------------------
 * What requests.py examples_from_input_dict + TensorServingClient._make_example_request build, serialised with
 * SerializeToString(deterministic=True).  ClassificationRequest and RegressionRequest share their field numbers (model_spec = 1,
 * input = 2), so one set of bytes serves both RPCs.  Row i of every column is example i, flattened in C order; the feature map of
 * every example lists the columns in `order` (B200TFS_ORDER_UPB: what deterministic serialisation gives).  Floating columns
 * (DT_FLOAT, DT_DOUBLE, DT_HALF) become float_list the way astype(float32) and a Python float make them: float32 signalling NaNs
 * quieted; float64 rounded to nearest even, NaN -> sign | 0x7FC00000 | (mantissa >> 29); float16 widened exactly, NaNs quieted.
 * Integer and bool columns become int64_list: sign-extended, uint64 wraps (2**64-1 is written as -1), a bool byte != 0 is 1.
 * A row of 0 elements still writes its empty list.  Strings (bytes_list) are taken as DT_STRING columns with a b200tfs_bytes
 * entry (the *_example_columns_* entry points, below); without one a DT_STRING column is B200TFS_E_DTYPE.
 * A variable-length (ragged) column is a padded one plus a b200tfs_ragged entry (the *_ragged entry points): row_elems is then the
 * padded row, and example i takes only the first lengths[i] * unit elements of its row.                                          */
typedef struct b200tfs_feature {
  const void* data;     /* n_examples rows of row_elems elements (one row with B200TFS_F_BROADCAST), C-contiguous, native order,
                           aligned to the element size; a DEVICE pointer for the _async entry point                              */
  int32_t src_dtype;    /* DT_FLOAT / DT_DOUBLE / DT_HALF / DT_INT8..64 / DT_UINT8..64 / DT_BOOL, DT_STRING with a b200tfs_bytes
                           entry; others: B200TFS_E_DTYPE                                                                        */
  uint32_t flags;       /* B200TFS_F_DEVICE_DATA (the _host entry point: `data` is in HBM already), B200TFS_F_BROADCAST           */
  int64_t row_elems;    /* elements per example (a ragged column: its padded row, max_len * unit)                              */
  const char* key;      /* feature name bytes (UTF-8, not NUL terminated)                                                       */
  int64_t key_len;
} b200tfs_feature;

typedef struct b200tfs_example_request {
  const char* model_name;
  int64_t model_name_len;
  int32_t has_version;  /* model_version is not None                                                                            */
  int32_t order;        /* B200TFS_ORDER_*: order of the features inside every example                                          */
  int64_t version;
  int64_t n_examples;   /* >= 0; an example has at least one feature                                                            */
  int32_t n_features;
  int32_t flags;        /* B200TFS_RF_GRPC_FRAME                                                                                */
  const b200tfs_feature* features;
} b200tfs_example_request;

/* Exact wire length (host, closed form) of a request without integer columns - replaces building the request with
 * requests.py examples_from_input_dict / _make_example_request and asking the message for ByteSize().  A request with an
 * integer column: B200TFS_E_ARG (its length depends on the values).  Over 2 GiB: B200TFS_E_TOOBIG.  This is the DENSE size:
 * it knows nothing of ragged lengths, so a caller with a ragged column sizes with b200tfs_example_arena_size instead.       */
int b200tfs_example_request_size(const b200tfs_example_request* r, uint64_t* total_len);
/* Arena bytes b200tfs_encode_example_requests_async needs: one 256-byte aligned slot per request, sized for its worst case
 * (10 bytes per integer element).  A request that cannot stay under 2 GiB whatever its values: B200TFS_E_TOOBIG.  It serves the
 * _ragged entry points unchanged: a ragged column is described by its padded row_elems, and that worst case bounds every length. */
int b200tfs_example_arena_size(int32_t n, const b200tfs_example_request* reqs, uint64_t* bytes);
/* Encode n requests from DEVICE columns into the device arena (256-byte aligned; b200tfs_example_arena_size bytes) - what
 * requests.py examples_from_input_dict + _make_example_request + SerializeToString(deterministic=True) produce.  Kernels only:
 * count (requests with an integer column: packed lengths and example sizes), scan (example offsets), emit (framing and values,
 * one contiguous range of examples and of wire per CTA), frame (the request prefix, written in front of the examples once
 * their total is known).  Never synchronises and is graph-capturable; a replay adapts to new integer values.  Collect rec_off /
 * rec_len with b200tfs_encode_results (a request over 2 GiB: B200TFS_E_TOOBIG).                                          */
int b200tfs_encode_example_requests_async(b200tfs_ctx* ctx, int32_t n, const b200tfs_example_request* reqs, void* arena_dev,
                                          uint64_t arena_cap);
/* The same from HOST columns (pinned or pageable; B200TFS_F_DEVICE_DATA columns are read in place): the columns are copied to
 * the device, encoded, and the records copied back into wire_host (capacity wire_cap: b200tfs_example_arena_size bytes are
 * always enough); rec_off / rec_len count from wire_host.  Synchronous.  Replaces requests.py examples_from_input_dict +
 * _make_example_request + SerializeToString.                                                                              */
int b200tfs_encode_example_requests_host(b200tfs_ctx* ctx, int32_t n, const b200tfs_example_request* reqs, void* wire_host,
                                         uint64_t wire_cap, uint64_t* rec_off, uint64_t* rec_len);

/* Variable-length columns (what a tf.Example model parses as VarLenFeature / RaggedFeature): one entry per feature of every
 * request, in request-then-feature order (the order of reqs[r].features), parallel to the features as b200tfs_pad_input is to the
 * inputs of a padded encode.  lengths == NULL: a dense column.  Otherwise feature.row_elems == max_len * unit (B200TFS_E_ARG
 * when not, when max_len or unit is negative, or on a B200TFS_F_BROADCAST feature) and example i's values are the first
 * lengths[i] * unit elements of its padded row; unit (the elements of one step of the ragged dimension) may be 0.         */
typedef struct b200tfs_ragged {
  const int64_t* lengths;   /* int64[n_examples], 8-byte aligned; device memory for the _async entry point                       */
  int64_t max_len;          /* L, the padded length                                                                               */
  int64_t unit;             /* elements per step of the ragged dimension (the product of the inner dims)                        */
  uint32_t flags;           /* B200TFS_F_DEVICE_DATA: the _host entry point finds the lengths in HBM already                      */
  int32_t pad_;
} b200tfs_ragged;
/* b200tfs_encode_example_requests_async with ragged columns (ragged == NULL: that call itself).  The lengths are only read on the
 * device, so a replayed CUDA graph follows whatever they hold then.  A length outside [0, max_len] gives that request
 * B200TFS_E_SHAPE in b200tfs_encode_results (rec_off = rec_len = 0); the kernels clamp it first, so no read leaves the padded
 * row and no write leaves the request's slot, and the other requests of the call are unaffected.                           */
int b200tfs_encode_example_requests_ragged_async(b200tfs_ctx* ctx, int32_t n, const b200tfs_example_request* reqs,
                                                 const b200tfs_ragged* ragged, void* arena_dev, uint64_t arena_cap);
/* b200tfs_encode_example_requests_host with ragged columns (ragged == NULL: that call itself).  Host lengths are copied to the
 * device with the columns, and checked on the host first (B200TFS_E_SHAPE before anything is launched).                      */
int b200tfs_encode_example_requests_ragged_host(b200tfs_ctx* ctx, int32_t n, const b200tfs_example_request* reqs,
                                                const b200tfs_ragged* ragged, void* wire_host, uint64_t wire_cap, uint64_t* rec_off,
                                                uint64_t* rec_len);

/* What message carries a request's examples: one entry per request, parallel to reqs (targets == NULL: every request LIST).
 *   B200TFS_EXAMPLES_LIST:           the ClassificationRequest / RegressionRequest above (key ignored).
 *   B200TFS_EXAMPLES_PREDICT_STRING: a PredictRequest with one input, `key`, a DT_STRING tensor of shape [n_examples] whose
 *                                    string_val holds every example serialised (the input of a model that runs tf.io.parse_example,
 *                                    e.g. a TFX or Estimator export's serving_default).  Its bytes are those of
 *                                    PredictRequest{model_spec, inputs[key] = TensorProto{dtype: DT_STRING, tensor_shape {dim {size:
 *                                    n}}, string_val: [e.SerializeToString(deterministic=True) for e in the examples]}}
 *                                    serialised with SerializeToString(deterministic=True); each example's bytes are exactly its
 *                                    bytes in the example_list.
 * A call may mix both, and B200TFS_EXAMPLES_PREDICT_ELWC (below), which needs a context.  An unknown kind, a negative key_len
 * or a NULL key with key_len > 0: B200TFS_E_ARG; a key over 2 GiB: B200TFS_E_TOOBIG - checked before the context is looked at. */
#define B200TFS_EXAMPLES_LIST 0
#define B200TFS_EXAMPLES_PREDICT_STRING 1
typedef struct b200tfs_example_target {
  int32_t kind;             /* B200TFS_EXAMPLES_*                                                                                 */
  int32_t pad_;
  const char* key;          /* PREDICT_STRING: the input's key bytes (UTF-8, not NUL terminated)                                  */
  int64_t key_len;
} b200tfs_example_target;
/* b200tfs_example_request_size, b200tfs_example_arena_size, b200tfs_encode_example_requests_ragged_async and
 * b200tfs_encode_example_requests_ragged_host with targets (target / targets == NULL: those calls themselves).                  */
int b200tfs_example_target_request_size(const b200tfs_example_request* r, const b200tfs_example_target* target, uint64_t* total_len);
int b200tfs_example_target_arena_size(int32_t n, const b200tfs_example_request* reqs, const b200tfs_example_target* targets,
                                      uint64_t* bytes);
int b200tfs_encode_example_targets_async(b200tfs_ctx* ctx, int32_t n, const b200tfs_example_request* reqs, const b200tfs_ragged* ragged,
                                         const b200tfs_example_target* targets, void* arena_dev, uint64_t arena_cap);
int b200tfs_encode_example_targets_host(b200tfs_ctx* ctx, int32_t n, const b200tfs_example_request* reqs, const b200tfs_ragged* ragged,
                                        const b200tfs_example_target* targets, void* wire_host, uint64_t wire_cap, uint64_t* rec_off,
                                        uint64_t* rec_len);

/* String columns (bytes_list), laid out as Arrow / cuDF hold them: one byte buffer and int64 offsets.  One entry per feature of
 * every request, in request-then-feature order, parallel to the features as b200tfs_ragged is.  offsets == NULL: not a bytes
 * column.  Otherwise the feature has src_dtype DT_STRING, `data` is the byte buffer (data_len bytes, any alignment) and row_elems
 * counts the strings of one example: string j is data[offsets[j], offsets[j+1]), the n_examples * row_elems strings (row_elems
 * with B200TFS_F_BROADCAST) fill the rows in order, and offsets[0] need not be 0 (a sliced column).  With a b200tfs_ragged entry
 * example i takes the first lengths[i] * unit strings of its padded row of max_len * unit.  Each string becomes one value of
 * the example's bytes_list; a row of no strings still writes its empty list.
 * The offsets of example i's row, starting at string b = i * row_elems (0 with B200TFS_F_BROADCAST), are read for its l_i
 * strings and for the next row's start, and must satisfy
 *     0 <= offsets[b] <= offsets[b+1] <= ... <= offsets[b + l_i] <= offsets[b + row_elems] <= data_len,
 * so that the rows are disjoint and in order: a request's strings take at most data_len bytes (n_examples * data_len broadcast),
 * which is what its arena slot is sized for.  Host offsets that break this: B200TFS_E_SHAPE before anything is launched.  Device
 * offsets are checked by the kernels: that request gets B200TFS_E_SHAPE in b200tfs_encode_results (rec_off = rec_len = 0), every
 * offset is clamped first, so no read leaves [data, data + data_len) and no write leaves the request's slot, and the other
 * requests of the call are unaffected.  A DT_STRING feature without an entry: B200TFS_E_DTYPE; an entry on another dtype, a
 * negative data_len, offsets not 8-byte aligned or unknown flags: B200TFS_E_ARG - checked before the context is looked at.      */
typedef struct b200tfs_bytes {
  const int64_t* offsets;   /* int64[strings + 1], 8-byte aligned; device memory for the _async entry point                      */
  int64_t data_len;         /* bytes of the buffer the offsets index (cuDF's int32 offsets must be widened to int64 first)      */
  uint32_t flags;           /* B200TFS_F_DEVICE_DATA: the _host entry point finds the offsets in HBM already (the data has its own
                               flag on the feature)                                                                              */
  int32_t pad_;
} b200tfs_bytes;
/* b200tfs_example_target_arena_size, b200tfs_encode_example_targets_async and b200tfs_encode_example_targets_host with bytes
 * columns (bytes == NULL: those calls themselves).  The slot of a request with a bytes column is sized from its data_len and
 * 11 bytes per string instead of a per-example worst case; the kernels count and place every example, and a replayed CUDA graph
 * follows whatever the data, offsets and lengths hold then.  Host data and offsets are copied to the device with the columns.   */
int b200tfs_example_columns_arena_size(int32_t n, const b200tfs_example_request* reqs, const b200tfs_bytes* bytes,
                                       const b200tfs_example_target* targets, uint64_t* bytes_out);
int b200tfs_encode_example_columns_async(b200tfs_ctx* ctx, int32_t n, const b200tfs_example_request* reqs, const b200tfs_ragged* ragged,
                                         const b200tfs_bytes* bytes, const b200tfs_example_target* targets, void* arena_dev,
                                         uint64_t arena_cap);
int b200tfs_encode_example_columns_host(b200tfs_ctx* ctx, int32_t n, const b200tfs_example_request* reqs, const b200tfs_ragged* ragged,
                                        const b200tfs_bytes* bytes, const b200tfs_example_target* targets, void* wire_host,
                                        uint64_t wire_cap, uint64_t* rec_off, uint64_t* rec_len);

/* A shared context (tensorflow.serving.ExampleListWithContext, Input field 2): one context Example for the whole request next to
 * its examples - the input of a ranking or recommendation model, whose per-query features then travel once instead of in every
 * candidate.  One entry per request, parallel to reqs (contexts == NULL: no request has one).  present == 0: the request is the
 * one the calls above encode.  present == 1:
 *   B200TFS_EXAMPLES_LIST:         the ClassificationRequest / RegressionRequest {model_spec, input {example_list_with_context
 *                                  {examples, context}}}, what requests.py examples_with_context_from_input_dict builds;
 *   B200TFS_EXAMPLES_PREDICT_ELWC: a PredictRequest whose one input `key` is a DT_STRING tensor of shape [1] whose string_val is
 *                                  that ExampleListWithContext serialised (TF-Ranking's serving input, one query per request):
 *                                  PredictRequest{model_spec, inputs[key] = TensorProto{dtype: DT_STRING, tensor_shape {dim {size:
 *                                  1}}, string_val: [elwc.SerializeToString(deterministic=True)]}}.
 * Both serialised with SerializeToString(deterministic=True); the ExampleListWithContext bytes are the same in both, and its
 * examples are those of the example_list.  The context Example's feature k holds all of context feature k's row_elems values
 * (`data` holds exactly one row; n_examples plays no part), converted as an example's are, listed in the request's `order`; a
 * context of no features is an empty Example (wire 12 00).  It comes after the examples on the wire:
 *     ... 12 vi(elwc) {0A vi(ex) ex}* 12 vi(ctx) 0A vi(F) entries
 * A context's DT_STRING features take b200tfs_bytes entries (context_bytes: one per feature of every present context, in
 * request-then-feature order) under the rule above with n_examples = 1; its slot grows by its worst case (10 bytes per integer
 * element, data_len + 11 per string).  Refused before the context is looked at: present not 0 or 1, a negative n_features, NULL
 * features with n_features > 0, a B200TFS_F_BROADCAST context feature, PREDICT_STRING with present == 1 and PREDICT_ELWC without
 * (B200TFS_E_ARG); a DT_STRING context feature without a bytes entry (B200TFS_E_DTYPE); host offsets that break the rule
 * (B200TFS_E_SHAPE, _host).  Device offsets of a context are checked by the kernels as an example's are: that request gets
 * B200TFS_E_SHAPE in b200tfs_encode_results, and no write leaves its slot.                                                   */
#define B200TFS_EXAMPLES_PREDICT_ELWC 2
typedef struct b200tfs_example_context {
  const b200tfs_feature* features;   /* host array; each feature's data is one row of row_elems values, placed as b200tfs_feature
                                        says for the entry point                                                                 */
  int32_t n_features;
  int32_t present;                   /* 0: no context; 1: this one (an empty one with n_features == 0)                            */
} b200tfs_example_context;
/* b200tfs_example_target_request_size with a context (context == NULL: that call itself): the exact length, in closed form,
 * when no integer or bytes column appears in the examples or the context (B200TFS_E_ARG otherwise).                          */
int b200tfs_example_context_request_size(const b200tfs_example_request* r, const b200tfs_example_target* target,
                                         const b200tfs_example_context* context, uint64_t* total_len);
/* b200tfs_example_columns_arena_size, b200tfs_encode_example_columns_async and b200tfs_encode_example_columns_host with contexts
 * (contexts == NULL: those calls themselves, which call these).  A call with contexts launches the count and scan kernels over
 * the contexts that have an integer or bytes column too, and its frame kernel writes each context behind its examples.         */
int b200tfs_example_context_arena_size(int32_t n, const b200tfs_example_request* reqs, const b200tfs_bytes* bytes,
                                       const b200tfs_example_target* targets, const b200tfs_example_context* contexts,
                                       const b200tfs_bytes* context_bytes, uint64_t* bytes_out);
int b200tfs_encode_example_contexts_async(b200tfs_ctx* ctx, int32_t n, const b200tfs_example_request* reqs, const b200tfs_ragged* ragged,
                                          const b200tfs_bytes* bytes, const b200tfs_example_target* targets,
                                          const b200tfs_example_context* contexts, const b200tfs_bytes* context_bytes, void* arena_dev,
                                          uint64_t arena_cap);
int b200tfs_encode_example_contexts_host(b200tfs_ctx* ctx, int32_t n, const b200tfs_example_request* reqs, const b200tfs_ragged* ragged,
                                         const b200tfs_bytes* bytes, const b200tfs_example_target* targets,
                                         const b200tfs_example_context* contexts, const b200tfs_bytes* context_bytes, void* wire_host,
                                         uint64_t wire_cap, uint64_t* rec_off, uint64_t* rec_len);

/* MultiInference (tensorflow.serving.MultiInferenceRequest, inference.proto): several Classify / Regress signatures of one model
 * over one Input.  One entry per request, parallel to reqs (tasks == NULL: no request has any).  n_tasks == 0: the request is the
 * one the calls above encode.  n_tasks > 0 (B200TFS_EXAMPLES_LIST only, with or without a context): a MultiInferenceRequest
 *     [00 be32(msg)] {0A vi(task) 0A vi(spec) <model_spec body> [1A vi(sig) sig] 12 vi(m) method}* 12 vi(input) <Input>
 * what SerializeToString(deterministic=True) writes: every task's model_spec is the request's (name, version) plus the task's
 * signature_name, its method_name "tensorflow/serving/classify" or "tensorflow/serving/regress"; the Input is the one the request
 * has without tasks (an example_list, or an ExampleListWithContext with a context).  The same kernels run.  Refused before the
 * context is looked at (B200TFS_E_ARG): n_tasks < 0, NULL tasks with n_tasks > 0, n_tasks > 0 with a PREDICT target kind, an
 * unknown method, a negative signature_len or a NULL signature_name with signature_len > 0.                                    */
typedef struct b200tfs_inference_task {
  const char* signature_name;  /* UTF-8, written as given                                                                       */
  int64_t signature_len;       /* 0: no signature_name field (the server's default signature)                                   */
  int32_t method;              /* B200TFS_RESP_CLASSIFY / B200TFS_RESP_REGRESS                                                  */
  int32_t pad_;
} b200tfs_inference_task;
typedef struct b200tfs_example_tasks {
  const b200tfs_inference_task* tasks;   /* host array of n_tasks                                                                */
  int32_t n_tasks;
  int32_t pad_;
} b200tfs_example_tasks;
/* b200tfs_example_context_request_size, _arena_size, b200tfs_encode_example_contexts_{async,host} with tasks (tasks == NULL: those
 * calls themselves, which call these).                                                                                          */
int b200tfs_example_tasks_request_size(const b200tfs_example_request* r, const b200tfs_example_target* target,
                                       const b200tfs_example_context* context, const b200tfs_example_tasks* tasks, uint64_t* total_len);
int b200tfs_example_tasks_arena_size(int32_t n, const b200tfs_example_request* reqs, const b200tfs_bytes* bytes,
                                     const b200tfs_example_target* targets, const b200tfs_example_context* contexts,
                                     const b200tfs_bytes* context_bytes, const b200tfs_example_tasks* tasks, uint64_t* bytes_out);
int b200tfs_encode_example_tasks_async(b200tfs_ctx* ctx, int32_t n, const b200tfs_example_request* reqs, const b200tfs_ragged* ragged,
                                       const b200tfs_bytes* bytes, const b200tfs_example_target* targets,
                                       const b200tfs_example_context* contexts, const b200tfs_bytes* context_bytes,
                                       const b200tfs_example_tasks* tasks, void* arena_dev, uint64_t arena_cap);
int b200tfs_encode_example_tasks_host(b200tfs_ctx* ctx, int32_t n, const b200tfs_example_request* reqs, const b200tfs_ragged* ragged,
                                      const b200tfs_bytes* bytes, const b200tfs_example_target* targets,
                                      const b200tfs_example_context* contexts, const b200tfs_bytes* context_bytes,
                                      const b200tfs_example_tasks* tasks, void* wire_host, uint64_t wire_cap, uint64_t* rec_off,
                                      uint64_t* rec_len);

/* SequenceExamples (tensorflow.SequenceExample, example.proto): the input of a model exported with a tf.io.parse_sequence_example
 * serving input - session and event-history models, TF-Ranking's SequenceExample format.  One entry per request, parallel to reqs
 * (sequences == NULL: no request has one).  present == 1 with target kind B200TFS_EXAMPLES_PREDICT_SEQUENCE: the request is
 *     PredictRequest{model_spec, inputs[key] = TensorProto{dtype: DT_STRING, tensor_shape {dim {size: n}}, string_val:
 *                    [s.SerializeToString(deterministic=True) for s in the n = n_examples sequences]}}
 * serialised with SerializeToString(deterministic=True) - the PREDICT_STRING prefix, sequences in place of examples:
 *     42 vi(S) 0A vi(C) {context map entries} 12 vi(G) {0A vi(e) 0A vi(klen) key 12 vi(FL) {0A vi(feat) Feature}*}*
 * The request's first n_context features are context features: sequence i's context holds them exactly as example i would (row
 * i, B200TFS_F_BROADCAST rows repeated, b200tfs_ragged and b200tfs_bytes entries as for an example), listed in `order`.  The
 * other features are feature lists, in `order` as well: each needs a b200tfs_ragged entry whose max_len is its step count T and
 * whose unit is the elements of one step (row_elems == T * unit).  With lengths == NULL every sequence has T steps, otherwise
 * sequence i has lengths[i] (a length outside [0, T] is B200TFS_E_SHAPE, host lengths before any launch, device ones in
 * b200tfs_encode_results).  Step t of sequence i is one Feature (a FeatureList entry, tag 0A) of elements [t * unit, (t + 1) *
 * unit) of row i, converted as an example's values are; a bytes list's row is strings [i * row_elems, (i + 1) * row_elems) under
 * the offsets rule of b200tfs_bytes with l_i = lengths[i] * unit.  A list of 0 steps still has its map entry, a step of 0
 * elements still writes its empty list, and a sequence of no features is 42 04 0A 00 12 00.  A call may mix sequence requests
 * with every other kind; sequence requests have their own count and emit kernels, and calls without one launch what they did.
 * Refused before the context is looked at (B200TFS_E_ARG): present not 0 or 1; present == 1 on another kind, PREDICT_SEQUENCE
 * without present == 1; a sequence request with a present context or with tasks; n_context outside [0, n_features]; a feature
 * list with B200TFS_F_BROADCAST, without a ragged entry (ragged == NULL), with a negative max_len or unit, unknown ragged flags,
 * unaligned lengths or row_elems != max_len * unit.  T over 2 GiB, or a request that cannot stay under 2 GiB: B200TFS_E_TOOBIG. */
#define B200TFS_EXAMPLES_PREDICT_SEQUENCE 3
typedef struct b200tfs_example_sequence {
  int32_t present;                   /* 0: not a sequence request; 1: one                                                        */
  int32_t n_context;                 /* features [0, n_context) of the request are context features, the rest feature lists      */
} b200tfs_example_sequence;
/* b200tfs_example_tasks_request_size with sequences (sequence == NULL: that call itself).  The exact length in closed form when no
 * integer or bytes column and no ragged entry with lengths appears in the request (B200TFS_E_ARG otherwise).                  */
int b200tfs_example_sequences_request_size(const b200tfs_example_request* r, const b200tfs_example_target* target,
                                           const b200tfs_example_context* context, const b200tfs_example_tasks* tasks,
                                           const b200tfs_ragged* ragged, const b200tfs_example_sequence* sequence, uint64_t* total_len);
/* b200tfs_example_tasks_arena_size with sequences and their ragged entries (both NULL: that call itself).  A sequence's slot takes
 * its worst case, whatever the values and lengths: T steps of each list, 10 bytes per integer element, data_len + 11 per
 * string, plus the step headers - so one captured graph serves any values, lengths and offsets.                             */
int b200tfs_example_sequences_arena_size(int32_t n, const b200tfs_example_request* reqs, const b200tfs_ragged* ragged,
                                         const b200tfs_bytes* bytes, const b200tfs_example_target* targets,
                                         const b200tfs_example_context* contexts, const b200tfs_bytes* context_bytes,
                                         const b200tfs_example_tasks* tasks, const b200tfs_example_sequence* sequences,
                                         uint64_t* bytes_out);
/* b200tfs_encode_example_tasks_{async,host} with sequences (sequences == NULL: those calls themselves, which call these).  A call
 * with a sequence request launches ex_seq_count_kernel over its sequences (one warp each: the context, then every step of every
 * list; an integer or bytes step's payload goes to a per-step scratch column sized from n and T alone), the unchanged scan over
 * every tile, and ex_emit_sequence_kernel over its spans; the frame kernel writes its prefix as PREDICT_STRING's.           */
int b200tfs_encode_example_sequences_async(b200tfs_ctx* ctx, int32_t n, const b200tfs_example_request* reqs, const b200tfs_ragged* ragged,
                                           const b200tfs_bytes* bytes, const b200tfs_example_target* targets,
                                           const b200tfs_example_context* contexts, const b200tfs_bytes* context_bytes,
                                           const b200tfs_example_tasks* tasks, const b200tfs_example_sequence* sequences,
                                           void* arena_dev, uint64_t arena_cap);
int b200tfs_encode_example_sequences_host(b200tfs_ctx* ctx, int32_t n, const b200tfs_example_request* reqs, const b200tfs_ragged* ragged,
                                          const b200tfs_bytes* bytes, const b200tfs_example_target* targets,
                                          const b200tfs_example_context* contexts, const b200tfs_bytes* context_bytes,
                                          const b200tfs_example_tasks* tasks, const b200tfs_example_sequence* sequences,
                                          void* wire_host, uint64_t wire_cap, uint64_t* rec_off, uint64_t* rec_len);
/* The _sequences_ entry points with a b200tfs_request_spec per request (spec / specs == NULL: those calls themselves, which call
 * these).  signature_name and version_label go into the model_spec of every target; a MultiInference task's model_spec is
 * name | version | the task's signature | label, and a signature_name for the whole request beside tasks is B200TFS_E_ARG.
 * output_filter exists only on the Predict forms (PREDICT_STRING, PREDICT_ELWC, PREDICT_SEQUENCE), where the frame kernel writes
 * it behind the examples (and the context); a filter on any other request is B200TFS_E_ARG.                                   */
int b200tfs_example_specs_request_size(const b200tfs_example_request* r, const b200tfs_example_target* target,
                                       const b200tfs_example_context* context, const b200tfs_example_tasks* tasks,
                                       const b200tfs_ragged* ragged, const b200tfs_example_sequence* sequence,
                                       const b200tfs_request_spec* spec, uint64_t* total_len);
int b200tfs_example_specs_arena_size(int32_t n, const b200tfs_example_request* reqs, const b200tfs_ragged* ragged,
                                     const b200tfs_bytes* bytes, const b200tfs_example_target* targets,
                                     const b200tfs_example_context* contexts, const b200tfs_bytes* context_bytes,
                                     const b200tfs_example_tasks* tasks, const b200tfs_example_sequence* sequences,
                                     const b200tfs_request_spec* specs, uint64_t* bytes_out);
int b200tfs_encode_example_specs_async(b200tfs_ctx* ctx, int32_t n, const b200tfs_example_request* reqs, const b200tfs_ragged* ragged,
                                       const b200tfs_bytes* bytes, const b200tfs_example_target* targets,
                                       const b200tfs_example_context* contexts, const b200tfs_bytes* context_bytes,
                                       const b200tfs_example_tasks* tasks, const b200tfs_example_sequence* sequences,
                                       const b200tfs_request_spec* specs, void* arena_dev, uint64_t arena_cap);
int b200tfs_encode_example_specs_host(b200tfs_ctx* ctx, int32_t n, const b200tfs_example_request* reqs, const b200tfs_ragged* ragged,
                                      const b200tfs_bytes* bytes, const b200tfs_example_target* targets,
                                      const b200tfs_example_context* contexts, const b200tfs_bytes* context_bytes,
                                      const b200tfs_example_tasks* tasks, const b200tfs_example_sequence* sequences,
                                      const b200tfs_request_spec* specs, void* wire_host, uint64_t wire_cap, uint64_t* rec_off,
                                      uint64_t* rec_len);

/* ---- Classify / Regress responses: a batch of responses into one value or score array ----------------------
 * What ClassificationResponse.FromString / RegressionResponse.FromString followed by a loop over the result give, concatenated
 * along the example axis across the n responses: row order is response 0's examples, then response 1's, and so on.
 *   B200TFS_RESP_REGRESS:  values float32[rows], values[row] = regressions[i].value.
 *   B200TFS_RESP_CLASSIFY: scores float32[rows * C] (row-major), scores[row * C + c] = classifications[i].classes[c].score, and
 *                          labels[row * C + c] = where that class's label lies, relative to its record.  C is the class count of
 *                          the batch's first example; every other example must have C classes too.
 * Floats come back as the runtime gives them: an absent score / value is +0.0, -0.0 stays -0.0, a signalling NaN is quieted.
 * Fields in any order, the last of repeated scalar fields wins, unknown fields (groups included) are skipped at every level, a
 * known field with another wire type is an unknown field, repeated `result` fields merge (their entries concatenate), repeated
 * model_spec fields merge.  Malformed wire - truncation, tag 0, a tag written in more than 5 bytes or past 32 bits, over-long
 * varints, lengths past the end, wire types 6 / 7, mismatched groups, a label or model_spec string that is not UTF-8 - is
 * B200TFS_E_PARSE, where FromString raises DecodeError.
 * One divergence: unknown groups nested more than 16 deep are B200TFS_E_PARSE here, while the runtime accepts them up to its
 * recursion limit of 100 (the message levels above the group included).  Codec.decode_*_responses send such a batch to the host
 * route, which gives the runtime's answer.                                                                                     */
#define B200TFS_RESP_REGRESS 1
#define B200TFS_RESP_CLASSIFY 2
typedef struct b200tfs_label_ref {
  uint32_t off;         /* label bytes, from the start of the record (0 / 0: the label is empty)                               */
  uint32_t len;
} b200tfs_label_ref;
/* Host only, closed form from the record lengths alone (every Regression, Classifications and Class entry takes at least two
 * bytes): *max_rows >= the rows of any responses of these lengths, *max_values >= their values (rows for Regress, rows * C for a
 * Classify batch that decodes).  Either pointer may be NULL.                                                                 */
int b200tfs_example_response_bound(int32_t kind, int32_t n, const uint64_t* rec_len, uint64_t* max_rows, uint64_t* max_values);
/* Decode n responses of `kind` lying at rec_off[i]..+rec_len[i] of the device arena.  values_dst (device) holds values_cap floats,
 * labels_dst (device; Classify only, may be NULL for Regress) labels_cap references.  Asynchronous and CUDA-graph capturable: the
 * kernels (index, scan, emit; Classify adds a label compare) find the rows on the device, so a graph captured once serves any
 * responses of the same lengths, and a replay adapts to new row counts.  Stores: values / labels of row r, class c < C only, and
 * never at or past values_cap / labels_cap; a response whose rows end past them is B200TFS_E_SIZE.  Collect the results with
 * b200tfs_example_response_results.                                                                                           */
int b200tfs_decode_example_responses(b200tfs_ctx* ctx, int32_t kind, const void* arena_dev, int32_t n, const uint64_t* rec_off,
                                     const uint64_t* rec_len, float* values_dst, uint64_t values_cap, b200tfs_label_ref* labels_dst,
                                     uint64_t labels_cap);
/* The same for responses in host memory (pinned for an asynchronous copy): the wire is copied to the device inside.  The
 * destinations are device memory as above.                                                                                   */
int b200tfs_decode_example_responses_host_async(b200tfs_ctx* ctx, int32_t kind, const void* wire_host, int32_t n,
                                                const uint64_t* rec_off, const uint64_t* rec_len, float* values_dst,
                                                uint64_t values_cap, b200tfs_label_ref* labels_dst, uint64_t labels_cap);
/* Results of the context's most recent b200tfs_decode_example_responses* call (synchronises); any pointer may be NULL.
 *   per_rec[3 * i + 0 .. 2]: the first row of response i, its rows, its status: B200TFS_OK, B200TFS_E_PARSE, B200TFS_E_SIZE (its
 *                            rows end past a capacity) or B200TFS_E_SHAPE (an example with another class count than C), in
 *                            that order of precedence.
 *   specs[i]:                its model_spec (offsets from the start of its record).
 *   batch[0 .. 4]:           rows of the batch, C (0 for Regress), same_labels (1: every example lists exactly the labels of the
 *                            first example, in the same order), the status of the first response that is not B200TFS_OK (or
 *                            B200TFS_OK), and that response's index (-1 when none).                                              */
int b200tfs_example_response_results(b200tfs_ctx* ctx, int32_t n, int64_t* per_rec, b200tfs_model_spec* specs, int64_t* batch);

/* ---- MultiInference responses: one value or score array per task ------------------------------------------------------------
 * n MultiInferenceResponses of a request with n_tasks tasks, kinds[t] (B200TFS_RESP_*) the method of task t.  TF Serving returns
 * one InferenceResult per task, in task order: task t's rows are those of results[t] across the n responses, decoded as the
 * Classify / Regress calls above decode a ClassificationResult / RegressionResult (C, labels and same_labels per task).  What
 * MultiInferenceResponse.FromString gives: each `results` field is its own result; inside one, model_spec fields merge, a oneof
 * member that occurs again merges (its entries concatenate), a different member clears the one before it; unknown fields and
 * groups are skipped at every level.  Per response and task, precedence as above: B200TFS_E_PARSE (malformed anywhere in the
 * response's results up to n_tasks; a malformed entry of a task's own result marks that task), B200TFS_E_SIZE, B200TFS_E_SHAPE
 * (a result count other than n_tasks - every task of the response -, a result whose member is not the one kinds[t] names - an
 * empty one included -, or an example with another class count than its task's C).  Tags and groups as above: a tag of more
 * than 5 bytes is B200TFS_E_PARSE, and so are unknown groups nested more than 16 deep, which the runtime accepts up to its
 * recursion limit of 100 (Codec.decode_multi_inference_responses sends those to the host route).
 * Host only, closed form: max_rows[t] / max_values[t] (n_tasks entries each; either may be NULL) bound task t as
 * b200tfs_example_response_bound does.                                                                                        */
int b200tfs_multi_inference_response_bound(int32_t n_tasks, const int32_t* kinds, int32_t n, const uint64_t* rec_len,
                                           uint64_t* max_rows, uint64_t* max_values);
/* Decode into values_dst[t] (device, values_cap[t] floats) and labels_dst[t] (device, labels_cap[t] references; Classify tasks
 * only, may be NULL) for every task t.  Asynchronous and CUDA-graph capturable: one index kernel (a warp per response) assigns
 * each result's entries to its task, then every task runs the scan, emit, [compare,] publish kernels of the Classify / Regress
 * decode.  Scratch is sized from n, n_tasks and the record lengths alone.  Stores as there, per task.                        */
int b200tfs_decode_multi_inference_responses(b200tfs_ctx* ctx, int32_t n_tasks, const int32_t* kinds, const void* arena_dev, int32_t n,
                                             const uint64_t* rec_off, const uint64_t* rec_len, float* const* values_dst,
                                             const uint64_t* values_cap, b200tfs_label_ref* const* labels_dst,
                                             const uint64_t* labels_cap);
int b200tfs_decode_multi_inference_responses_host_async(b200tfs_ctx* ctx, int32_t n_tasks, const int32_t* kinds, const void* wire_host,
                                                        int32_t n, const uint64_t* rec_off, const uint64_t* rec_len,
                                                        float* const* values_dst, const uint64_t* values_cap,
                                                        b200tfs_label_ref* const* labels_dst, const uint64_t* labels_cap);
/* Results of the most recent b200tfs_decode_multi_inference_responses* call (synchronises), task after task: per_rec[3 * (t * n +
 * i) + 0 .. 2], specs[t * n + i] (the model_spec of response i's result t) and batch[5 * t + 0 .. 4], each as
 * b200tfs_example_response_results gives them.                                                                               */
int b200tfs_multi_inference_response_results(b200tfs_ctx* ctx, int32_t n, int32_t n_tasks, int64_t* per_rec, b200tfs_model_spec* specs,
                                             int64_t* batch);

#ifdef __cplusplus
}
#endif
#endif /* B200TFS_H_ */
