"""ctypes binding of ``libb200tfs.so`` (C ABI declared in ``include/b200tfs.h``).

No PyTorch and no CUDA Python package: the shared library is the only native dependency, loaded from
``min-tfs-client_b200/lib/``.  If the library is missing or no CUDA device is present the codec fails
loudly (``RuntimeError``) - there is no CPU fallback behind this module.
"""
from __future__ import annotations

import ctypes as C
import os
import threading

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("B200TFS_LIB") or os.path.join(os.path.dirname(_HERE), "lib", "libb200tfs.so")   # B200TFS_LIB: experiment builds

# ---- status codes (b200tfs.h) -----------------------------------------------------------------
OK = 0
E_DTYPE, E_SHAPE, E_SIZE, E_PARSE, E_CUDA, E_TOOBIG, E_ARG, E_NONCANONICAL, E_RANGE, E_KEY, E_SPILL = range(-1, -12, -1)

F_TENSOR_CONTENT = 0x1
F_KEEP_SNAN = 0x2
F_PRESERIALIZED = 0x4
F_DEVICE_DATA = 0x8
RF_GRPC_FRAME = 0x1
OF_TENSOR_CONTENT, OF_MULTI_CHUNK, OF_DIM_INFERRED, OF_HAS_UNKNOWN, OF_RANK0, OF_VARINT, OF_PAD_EDGE = 0x1, 0x2, 0x4, 0x8, 0x10, 0x20, 0x40
OF_UNPACKED, OF_SPILLED, OF_DEVICE_VARINT = 0x80, 0x100, 0x200
ORDER_GIVEN, ORDER_UPB, ORDER_BYTES = 0, 1, 2
MAX_RANK, MAX_RUNS, FUSED_MAX_OUTPUTS, CONCAT_MAX_KEYS = 16, 8, 8, 8
DT_HALF_REFQUIRK = -19


class NativeError(RuntimeError):
    """A non-OK status from libb200tfs that has no closer Python exception type."""

    def __init__(self, code, message):
        super().__init__(f"libb200tfs error {code}: {message}")
        self.code = code


class Tensor(C.Structure):
    _fields_ = [
        ("data", C.c_void_p), ("src_dtype", C.c_int32), ("wire_dtype", C.c_int32), ("rank", C.c_int32),
        ("flags", C.c_uint32), ("dims", C.POINTER(C.c_int64)), ("key", C.c_char_p), ("key_len", C.c_int64),
        ("packed_len", C.c_uint64),
    ]


class Request(C.Structure):
    _fields_ = [
        ("model_name", C.c_char_p), ("model_name_len", C.c_int64), ("has_version", C.c_int32), ("order", C.c_int32),
        ("version", C.c_int64), ("n_inputs", C.c_int32), ("flags", C.c_int32), ("inputs", C.POINTER(Tensor)),
    ]


class RequestSpec(C.Structure):
    """b200tfs_request_spec: a request's ModelSpec.signature_name (signature_len 0: not written), ModelSpec.version_label
    (version_label_len < 0: not set) and PredictRequest.output_filter (n_output_filter names), for the ``_spec`` entry points."""
    _fields_ = [
        ("signature_name", C.c_char_p), ("signature_len", C.c_int64), ("version_label", C.c_char_p), ("version_label_len", C.c_int64),
        ("output_filter", C.POINTER(C.c_char_p)), ("output_filter_len", C.POINTER(C.c_int64)), ("n_output_filter", C.c_int64),
    ]


class Run(C.Structure):
    """b200tfs_run: `count` pieces of `len` value bytes, `stride` bytes apart, from TensorProto field `field`."""
    _fields_ = [("off", C.c_uint64), ("len", C.c_uint32), ("count", C.c_uint32), ("stride", C.c_uint32), ("field", C.c_uint32)]


class Output(C.Structure):
    _fields_ = [
        ("key_off", C.c_uint64), ("key_len", C.c_uint32), ("dtype", C.c_int32), ("rank", C.c_int32), ("flags", C.c_uint32),
        ("value_field", C.c_int32), ("n_runs", C.c_int32), ("dims", C.c_int64 * MAX_RANK),
        ("runs", Run * MAX_RUNS),
        ("content_off", C.c_uint64), ("content_len", C.c_uint64), ("msg_off", C.c_uint64), ("msg_len", C.c_uint64),
        ("n_elems", C.c_uint64), ("dst_bytes", C.c_uint64), ("n_strings", C.c_uint64), ("dst_off", C.c_uint64), ("status", C.c_int32),
        ("n_inline", C.c_uint32), ("spill_rec", C.c_uint32), ("spill_seq", C.c_uint32),
    ]


class ModelSpec(C.Structure):
    _fields_ = [
        ("name_off", C.c_uint64), ("name_len", C.c_uint32), ("signature_len", C.c_uint32), ("signature_off", C.c_uint64),
        ("label_off", C.c_uint64), ("label_len", C.c_uint32), ("has_version", C.c_int32), ("version", C.c_int64),
    ]


class ConcatKey(C.Structure):
    """b200tfs_concat_key: one requested output of b200tfs_decode_concat (in: key, dst, dst_cap; out: the layout)."""
    _fields_ = [
        ("key", C.c_char_p), ("key_len", C.c_int64), ("dst", C.c_void_p), ("dst_cap", C.c_uint64), ("dtype", C.c_int32),
        ("rank", C.c_int32), ("dims", C.c_int64 * MAX_RANK), ("bytes", C.c_uint64), ("status", C.c_int32), ("bad_rec", C.c_int32),
    ]


class ConcatStrings(C.Structure):
    """b200tfs_concat_strings: the byte buffer of one DT_STRING key of b200tfs_decode_concat_strings, whose int64 offsets go to the
    key's dst (in: data, data_cap; out of b200tfs_concat_strings_layout: strings, data_bytes)."""
    _fields_ = [("data", C.c_void_p), ("data_cap", C.c_uint64), ("strings", C.c_uint64), ("data_bytes", C.c_uint64)]


class PadKey(C.Structure):
    """b200tfs_pad_key: one requested output of b200tfs_decode_padded (in: key, dst, dst_cap, rank, dims[1:], pad_bits; out: the
    layout)."""
    _fields_ = [
        ("key", C.c_char_p), ("key_len", C.c_int64), ("dst", C.c_void_p), ("dst_cap", C.c_uint64), ("dtype", C.c_int32),
        ("rank", C.c_int32), ("dims", C.c_int64 * MAX_RANK), ("bytes", C.c_uint64), ("status", C.c_int32), ("bad_rec", C.c_int32),
        ("pad_bits", C.c_uint8 * 16),
    ]


class PaddedStrings(C.Structure):
    """b200tfs_padded_strings: the byte buffer and pad string of one DT_STRING key of b200tfs_decode_padded_strings, whose int64
    offsets go to the key's dst (in: data, data_cap, pad, pad_len; out of b200tfs_padded_strings_layout: strings, data_bytes)."""
    _fields_ = [("data", C.c_void_p), ("data_cap", C.c_uint64), ("pad", C.c_void_p), ("pad_len", C.c_uint64), ("strings", C.c_uint64),
                ("data_bytes", C.c_uint64)]


F_BROADCAST = 0x10


class Feature(C.Structure):
    """b200tfs_feature: one column of a tf.Example request (row i is example i; F_BROADCAST: one row for every example)."""
    _fields_ = [
        ("data", C.c_void_p), ("src_dtype", C.c_int32), ("flags", C.c_uint32), ("row_elems", C.c_int64), ("key", C.c_char_p),
        ("key_len", C.c_int64),
    ]


class ExampleRequest(C.Structure):
    """b200tfs_example_request: one ClassificationRequest / RegressionRequest built from columns."""
    _fields_ = [
        ("model_name", C.c_char_p), ("model_name_len", C.c_int64), ("has_version", C.c_int32), ("order", C.c_int32),
        ("version", C.c_int64), ("n_examples", C.c_int64), ("n_features", C.c_int32), ("flags", C.c_int32),
        ("features", C.POINTER(Feature)),
    ]


class Ragged(C.Structure):
    """b200tfs_ragged: the lengths of one variable-length tf.Example column (NULL lengths: a dense column); example i takes the
    first lengths[i] * unit of its row's max_len * unit elements."""
    _fields_ = [("lengths", C.c_void_p), ("max_len", C.c_int64), ("unit", C.c_int64), ("flags", C.c_uint32), ("pad_", C.c_int32)]


class Bytes(C.Structure):
    """b200tfs_bytes: the int64 offsets of one string (bytes_list) tf.Example column (NULL offsets: not a bytes column); string j
    is data[offsets[j]:offsets[j+1]] of the feature's byte buffer of data_len bytes."""
    _fields_ = [("offsets", C.c_void_p), ("data_len", C.c_int64), ("flags", C.c_uint32), ("pad_", C.c_int32)]


EXAMPLES_LIST, EXAMPLES_PREDICT_STRING, EXAMPLES_PREDICT_ELWC, EXAMPLES_PREDICT_SEQUENCE, EXAMPLES_PREDICT_ELWCS = 0, 1, 2, 3, 4


class ExampleTarget(C.Structure):
    """b200tfs_example_target: what carries one request's examples - a ClassificationRequest / RegressionRequest (EXAMPLES_LIST)
    or a PredictRequest whose input ``key`` is a DT_STRING vector of the serialized examples (EXAMPLES_PREDICT_STRING)."""
    _fields_ = [("kind", C.c_int32), ("pad_", C.c_int32), ("key", C.c_char_p), ("key_len", C.c_int64)]


class ExampleContext(C.Structure):
    """b200tfs_example_context: one request's shared context Example (present 0: none; 1: ``features``, each one row of all
    its values), which makes the request an ExampleListWithContext (EXAMPLES_LIST / EXAMPLES_PREDICT_ELWC)."""
    _fields_ = [("features", C.POINTER(Feature)), ("n_features", C.c_int32), ("present", C.c_int32)]


class InferenceTask(C.Structure):
    """b200tfs_inference_task: one task of a MultiInferenceRequest - a signature (signature_len 0: the server's default) run with
    the method RESP_CLASSIFY or RESP_REGRESS."""
    _fields_ = [("signature_name", C.c_char_p), ("signature_len", C.c_int64), ("method", C.c_int32), ("pad_", C.c_int32)]


class ExampleTasks(C.Structure):
    """b200tfs_example_tasks: the tasks of one request (n_tasks 0: not a MultiInferenceRequest)."""
    _fields_ = [("tasks", C.c_void_p), ("n_tasks", C.c_int32), ("pad_", C.c_int32)]


class ExampleSequence(C.Structure):
    """b200tfs_example_sequence: one request's SequenceExamples (present 0: none; 1: its first ``n_context`` features are
    context features, the rest feature lists whose Ragged entries give their steps), for EXAMPLES_PREDICT_SEQUENCE."""
    _fields_ = [("present", C.c_int32), ("n_context", C.c_int32)]


class ExampleLists(C.Structure):
    """b200tfs_example_lists: one request's queries for EXAMPLES_PREDICT_ELWCS (present 0: none; 1: ``n_lists`` ELWCs whose
    examples are the next ``list_sizes[q]`` rows, and whose contexts are row q of the ``n_context`` ``context`` features)."""
    _fields_ = [("list_sizes", C.c_void_p), ("n_lists", C.c_int64), ("context", C.POINTER(Feature)), ("n_context", C.c_int32),
                ("present", C.c_int32)]


class ExampleDeviceLists(C.Structure):
    """b200tfs_example_device_lists: one request's list sizes in device memory (``sizes``: a device int64[n_lists]; None: the
    host ``list_sizes`` of its ExampleLists entry, or not an EXAMPLES_PREDICT_ELWCS request)."""
    _fields_ = [("sizes", C.c_void_p)]


class PadInput(C.Structure):
    """b200tfs_pad_input: the shapes of one input of b200tfs_encode_padded_requests_async (int64[n, cols]; cols 1: row counts)."""
    _fields_ = [("shapes", C.c_void_p), ("cols", C.c_int32), ("pad_", C.c_int32)]


RESP_REGRESS, RESP_CLASSIFY = 1, 2


class LabelRef(C.Structure):
    """b200tfs_label_ref: a Class label's bytes, from the start of its record."""
    _fields_ = [("off", C.c_uint32), ("len", C.c_uint32)]


_u64p = C.POINTER(C.c_uint64)
_i32p = C.POINTER(C.c_int32)
_vp = C.c_void_p
_vpp = C.POINTER(C.c_void_p)

# every symbol include/b200tfs.h declares: name -> (restype, argtypes)
SIGNATURES = {
    "b200tfs_abi_version": (C.c_int, []),
    "b200tfs_last_error": (C.c_char_p, []),
    "b200tfs_device_count": (C.c_int, [_i32p]),
    "b200tfs_create": (C.c_int, [C.c_int, _vpp]),
    "b200tfs_destroy": (C.c_int, [_vp]),
    "b200tfs_sync": (C.c_int, [_vp]),
    "b200tfs_stream": (C.c_void_p, [_vp]),
    "b200tfs_set_stream": (C.c_int, [_vp, _vp]),
    "b200tfs_kernel_launches": (C.c_int, [_vp, _u64p]),
    "b200tfs_malloc": (C.c_int, [_vp, C.c_uint64, _vpp]),
    "b200tfs_free": (C.c_int, [_vp, _vp]),
    "b200tfs_host_alloc": (C.c_int, [C.c_uint64, _vpp]),
    "b200tfs_host_free": (C.c_int, [_vp]),
    "b200tfs_memcpy_h2d": (C.c_int, [_vp, _vp, _vp, C.c_uint64]),
    "b200tfs_memcpy_d2h": (C.c_int, [_vp, _vp, _vp, C.c_uint64]),
    "b200tfs_memcpy_d2d": (C.c_int, [_vp, _vp, _vp, C.c_uint64]),
    "b200tfs_memset": (C.c_int, [_vp, _vp, C.c_int, C.c_uint64]),
    "b200tfs_event_create": (C.c_int, [_vpp]),
    "b200tfs_event_destroy": (C.c_int, [_vp]),
    "b200tfs_event_record": (C.c_int, [_vp, _vp]),
    "b200tfs_event_sync": (C.c_int, [_vp]),
    "b200tfs_event_elapsed_ms": (C.c_int, [_vp, _vp, C.POINTER(C.c_float)]),
    "b200tfs_dtype_size": (C.c_int, [C.c_int32]),
    "b200tfs_dtype_field": (C.c_int, [C.c_int32]),
    "b200tfs_cast_supported": (C.c_int, [C.c_int32, C.c_int32]),
    "b200tfs_tensor_proto_size": (C.c_int, [C.POINTER(Tensor), _u64p, _u64p]),
    "b200tfs_request_size": (C.c_int, [C.POINTER(Request), _u64p]),
    "b200tfs_tensor_proto_header": (C.c_int, [C.POINTER(Tensor), _vp, C.c_uint64, _u64p]),
    "b200tfs_request_frame": (C.c_int, [C.POINTER(Request), _vp, C.c_uint64, _u64p, _u64p, _u64p, _i32p]),
    "b200tfs_order_keys": (C.c_int, [C.c_int32, C.POINTER(C.c_char_p), C.POINTER(C.c_int64), C.c_int32, _i32p]),
    "b200tfs_tensor_arena_size": (C.c_int, [C.c_int32, C.POINTER(Tensor), _u64p]),
    "b200tfs_request_arena_size": (C.c_int, [C.c_int32, C.POINTER(Request), _u64p]),
    "b200tfs_request_size_spec": (C.c_int, [C.POINTER(Request), C.POINTER(RequestSpec), _u64p]),
    "b200tfs_request_frame_spec": (C.c_int, [C.POINTER(Request), C.POINTER(RequestSpec), _vp, C.c_uint64, _u64p, _u64p, _u64p, _i32p]),
    "b200tfs_request_arena_size_spec": (C.c_int, [C.c_int32, C.POINTER(Request), C.POINTER(RequestSpec), _u64p]),
    "b200tfs_measure": (C.c_int, [_vp, C.c_int32, C.POINTER(Tensor)]),
    "b200tfs_encode_tensor_protos": (C.c_int, [_vp, C.c_int32, C.POINTER(Tensor), _vp, C.c_uint64, _u64p, _u64p]),
    "b200tfs_encode_requests": (C.c_int, [_vp, C.c_int32, C.POINTER(Request), _vp, C.c_uint64, _u64p, _u64p]),
    "b200tfs_encode_requests_async": (C.c_int, [_vp, C.c_int32, C.POINTER(Request), _vp, C.c_uint64]),
    "b200tfs_encode_results": (C.c_int, [_vp, C.c_int32, _u64p, _u64p]),
    "b200tfs_request_frame_deferred": (C.c_int, [C.POINTER(Request), _u64p, _vp, C.c_uint64, _u64p, _u64p, _u64p, _u64p]),
    "b200tfs_encode_requests_async_spec": (C.c_int, [_vp, C.c_int32, C.POINTER(Request), C.POINTER(RequestSpec), _vp, C.c_uint64]),
    "b200tfs_request_frame_deferred_spec": (C.c_int, [C.POINTER(Request), C.POINTER(RequestSpec), _u64p, _vp, C.c_uint64, _u64p, _u64p,
                                                      _u64p, _u64p]),
    "b200tfs_parse_responses": (C.c_int, [_vp, _vp, C.c_int32, _u64p, _u64p, C.c_int32, C.POINTER(Output), _i32p,
                                          C.POINTER(ModelSpec), _i32p]),
    "b200tfs_parse_tensor_protos": (C.c_int, [_vp, _vp, C.c_int32, _u64p, _u64p, C.POINTER(Output), _i32p]),
    "b200tfs_output_dims": (C.c_int, [_vp, C.POINTER(Output), C.POINTER(C.c_int64), C.c_int32]),
    "b200tfs_output_runs": (C.c_int, [_vp, C.POINTER(Output), C.POINTER(Run), C.c_int32]),
    "b200tfs_unpack_outputs": (C.c_int, [_vp, _vp, C.c_int32, C.POINTER(Output), _u64p, _vpp, _i32p, _i32p]),
    "b200tfs_decode_responses": (C.c_int, [_vp, _vp, C.c_int32, _u64p, _u64p, _vp, C.c_uint64]),
    "b200tfs_decode_results": (C.c_int, [_vp, C.c_int32, C.POINTER(Output), _i32p, C.POINTER(ModelSpec), _i32p]),
    "b200tfs_decode_stats": (C.c_int, [_vp, _u64p, _u64p, _u64p]),
    "b200tfs_concat_layout": (C.c_int, [_vp, C.c_int32, _u64p, _u64p, C.c_int32, C.POINTER(ConcatKey), C.c_int32]),
    "b200tfs_response_keys": (C.c_int, [_vp, C.c_uint64, C.c_int32, _u64p, C.POINTER(C.c_uint32), _i32p]),
    "b200tfs_decode_concat": (C.c_int, [_vp, _vp, C.c_int32, _u64p, _u64p, C.c_int32, C.POINTER(ConcatKey)]),
    "b200tfs_decode_concat_host_async": (C.c_int, [_vp, _vp, C.c_int32, _u64p, _u64p, C.c_int32, C.POINTER(ConcatKey)]),
    "b200tfs_concat_results": (C.c_int, [_vp, C.c_int32, C.c_int32, C.POINTER(Output), C.POINTER(ModelSpec), _i32p]),
    "b200tfs_concat_strings_layout": (C.c_int, [_vp, C.c_int32, _u64p, _u64p, C.c_int32, C.POINTER(ConcatKey), C.POINTER(ConcatStrings),
                                                C.c_int32]),
    "b200tfs_concat_strings_bound": (C.c_int, [C.c_int32, _u64p, _u64p, _u64p]),
    "b200tfs_decode_concat_strings": (C.c_int, [_vp, _vp, C.c_int32, _u64p, _u64p, C.c_int32, C.POINTER(ConcatKey),
                                                C.POINTER(ConcatStrings)]),
    "b200tfs_decode_concat_strings_host_async": (C.c_int, [_vp, _vp, C.c_int32, _u64p, _u64p, C.c_int32, C.POINTER(ConcatKey),
                                                           C.POINTER(ConcatStrings)]),
    "b200tfs_padded_layout": (C.c_int, [_vp, C.c_int32, _u64p, _u64p, C.c_int32, C.POINTER(PadKey), C.c_int32]),
    "b200tfs_decode_padded": (C.c_int, [_vp, _vp, C.c_int32, _u64p, _u64p, C.c_int32, C.POINTER(PadKey)]),
    "b200tfs_decode_padded_host_async": (C.c_int, [_vp, _vp, C.c_int32, _u64p, _u64p, C.c_int32, C.POINTER(PadKey)]),
    "b200tfs_padded_results": (C.c_int, [_vp, C.c_int32, C.c_int32, C.POINTER(Output), C.POINTER(ModelSpec), _i32p]),
    "b200tfs_padded_strings_layout": (C.c_int, [_vp, C.c_int32, _u64p, _u64p, C.c_int32, C.POINTER(PadKey), C.POINTER(PaddedStrings),
                                                C.c_int32]),
    "b200tfs_decode_padded_strings": (C.c_int, [_vp, _vp, C.c_int32, _u64p, _u64p, C.c_int32, C.POINTER(PadKey),
                                                C.POINTER(PaddedStrings)]),
    "b200tfs_decode_padded_strings_host_async": (C.c_int, [_vp, _vp, C.c_int32, _u64p, _u64p, C.c_int32, C.POINTER(PadKey),
                                                           C.POINTER(PaddedStrings)]),
    "b200tfs_padded_request_arena_size": (C.c_int, [C.c_int32, C.POINTER(Request), _u64p]),
    "b200tfs_encode_padded_requests_async": (C.c_int, [_vp, C.c_int32, C.POINTER(Request), C.POINTER(PadInput), _vp, C.c_uint64]),
    "b200tfs_padded_request_frame": (C.c_int, [C.POINTER(Request), C.POINTER(PadInput), _u64p, _vp, C.c_uint64, _u64p, _u64p, _u64p]),
    "b200tfs_padded_request_columns_arena_size": (C.c_int, [C.c_int32, C.POINTER(Request), C.POINTER(Bytes), _u64p]),
    "b200tfs_encode_padded_requests_columns_async": (C.c_int, [_vp, C.c_int32, C.POINTER(Request), C.POINTER(PadInput), C.POINTER(Bytes),
                                                               _vp, C.c_uint64]),
    "b200tfs_padded_request_frame_columns": (C.c_int, [C.POINTER(Request), C.POINTER(PadInput), C.POINTER(Bytes), _u64p, _vp, C.c_uint64,
                                                       _u64p, _u64p, _u64p]),
    "b200tfs_padded_request_columns_arena_size_spec": (C.c_int, [C.c_int32, C.POINTER(Request), C.POINTER(Bytes), C.POINTER(RequestSpec),
                                                                 _u64p]),
    "b200tfs_encode_padded_requests_columns_async_spec": (C.c_int, [_vp, C.c_int32, C.POINTER(Request), C.POINTER(PadInput),
                                                                    C.POINTER(Bytes), C.POINTER(RequestSpec), _vp, C.c_uint64]),
    "b200tfs_padded_request_frame_columns_spec": (C.c_int, [C.POINTER(Request), C.POINTER(PadInput), C.POINTER(Bytes),
                                                            C.POINTER(RequestSpec), _u64p, _vp, C.c_uint64, _u64p, _u64p, _u64p]),
    "b200tfs_capture_begin": (C.c_int, [_vp]),
    "b200tfs_capture_end": (C.c_int, [_vp, _vpp]),
    "b200tfs_graph_launch": (C.c_int, [_vp, _vp]),
    "b200tfs_graph_destroy": (C.c_int, [_vp]),
    "b200tfs_wait_event": (C.c_int, [_vp, _vp]),
    "b200tfs_encode_requests_host": (C.c_int, [_vp, C.c_int32, C.POINTER(Request), _vp, C.c_uint64, _u64p, _u64p]),
    "b200tfs_encode_requests_host_async": (C.c_int, [_vp, C.c_int32, C.POINTER(Request), _vp, C.c_uint64, _u64p, _u64p]),
    "b200tfs_encode_requests_host_spec": (C.c_int, [_vp, C.c_int32, C.POINTER(Request), C.POINTER(RequestSpec), _vp, C.c_uint64, _u64p,
                                                    _u64p]),
    "b200tfs_pipelined_calls": (C.c_int, [_vp, _u64p]),
    "b200tfs_direct_calls": (C.c_int, [_vp, _u64p]),
    "b200tfs_set_pipeline": (C.c_int, [_vp, C.c_uint64, C.c_int32]),
    "b200tfs_set_decode_cast": (C.c_int, [_vp, C.c_int32]),
    "b200tfs_set_decode_varints": (C.c_int, [_vp, C.c_int32]),
    "b200tfs_decode_slot_bytes": (C.c_int, [_vp, C.c_int32, _u64p, _u64p, C.c_int32, _u64p, _i32p]),
    "b200tfs_decode_responses_host_async": (C.c_int, [_vp, _vp, C.c_int32, _u64p, _u64p, _vp, C.c_uint64]),
    "b200tfs_encode_tensor_protos_host": (C.c_int, [_vp, C.c_int32, C.POINTER(Tensor), _vp, C.c_uint64, _u64p, _u64p]),
    "b200tfs_parse_responses_host": (C.c_int, [_vp, _vp, C.c_int32, _u64p, _u64p, C.c_int32, C.POINTER(Output), _i32p,
                                               C.POINTER(ModelSpec), _i32p]),
    "b200tfs_parse_tensor_protos_host": (C.c_int, [_vp, _vp, C.c_int32, _u64p, _u64p, C.POINTER(Output), _i32p]),
    "b200tfs_unpack_outputs_host": (C.c_int, [_vp, C.c_int32, C.POINTER(Output), _u64p, _vpp, _i32p, _i32p]),
    "b200tfs_example_request_size": (C.c_int, [C.POINTER(ExampleRequest), _u64p]),
    "b200tfs_example_arena_size": (C.c_int, [C.c_int32, C.POINTER(ExampleRequest), _u64p]),
    "b200tfs_encode_example_requests_async": (C.c_int, [_vp, C.c_int32, C.POINTER(ExampleRequest), _vp, C.c_uint64]),
    "b200tfs_encode_example_requests_host": (C.c_int, [_vp, C.c_int32, C.POINTER(ExampleRequest), _vp, C.c_uint64, _u64p, _u64p]),
    "b200tfs_encode_example_requests_ragged_async": (C.c_int, [_vp, C.c_int32, C.POINTER(ExampleRequest), C.POINTER(Ragged), _vp,
                                                               C.c_uint64]),
    "b200tfs_encode_example_requests_ragged_host": (C.c_int, [_vp, C.c_int32, C.POINTER(ExampleRequest), C.POINTER(Ragged), _vp,
                                                              C.c_uint64, _u64p, _u64p]),
    "b200tfs_example_target_request_size": (C.c_int, [C.POINTER(ExampleRequest), C.POINTER(ExampleTarget), _u64p]),
    "b200tfs_example_target_arena_size": (C.c_int, [C.c_int32, C.POINTER(ExampleRequest), C.POINTER(ExampleTarget), _u64p]),
    "b200tfs_encode_example_targets_async": (C.c_int, [_vp, C.c_int32, C.POINTER(ExampleRequest), C.POINTER(Ragged),
                                                       C.POINTER(ExampleTarget), _vp, C.c_uint64]),
    "b200tfs_encode_example_targets_host": (C.c_int, [_vp, C.c_int32, C.POINTER(ExampleRequest), C.POINTER(Ragged),
                                                      C.POINTER(ExampleTarget), _vp, C.c_uint64, _u64p, _u64p]),
    "b200tfs_example_columns_arena_size": (C.c_int, [C.c_int32, C.POINTER(ExampleRequest), C.POINTER(Bytes), C.POINTER(ExampleTarget),
                                                     _u64p]),
    "b200tfs_encode_example_columns_async": (C.c_int, [_vp, C.c_int32, C.POINTER(ExampleRequest), C.POINTER(Ragged), C.POINTER(Bytes),
                                                       C.POINTER(ExampleTarget), _vp, C.c_uint64]),
    "b200tfs_encode_example_columns_host": (C.c_int, [_vp, C.c_int32, C.POINTER(ExampleRequest), C.POINTER(Ragged), C.POINTER(Bytes),
                                                      C.POINTER(ExampleTarget), _vp, C.c_uint64, _u64p, _u64p]),
    "b200tfs_example_context_request_size": (C.c_int, [C.POINTER(ExampleRequest), C.POINTER(ExampleTarget), C.POINTER(ExampleContext),
                                                       _u64p]),
    "b200tfs_example_context_arena_size": (C.c_int, [C.c_int32, C.POINTER(ExampleRequest), C.POINTER(Bytes), C.POINTER(ExampleTarget),
                                                     C.POINTER(ExampleContext), C.POINTER(Bytes), _u64p]),
    "b200tfs_encode_example_contexts_async": (C.c_int, [_vp, C.c_int32, C.POINTER(ExampleRequest), C.POINTER(Ragged), C.POINTER(Bytes),
                                                        C.POINTER(ExampleTarget), C.POINTER(ExampleContext), C.POINTER(Bytes), _vp,
                                                        C.c_uint64]),
    "b200tfs_encode_example_contexts_host": (C.c_int, [_vp, C.c_int32, C.POINTER(ExampleRequest), C.POINTER(Ragged), C.POINTER(Bytes),
                                                       C.POINTER(ExampleTarget), C.POINTER(ExampleContext), C.POINTER(Bytes), _vp,
                                                       C.c_uint64, _u64p, _u64p]),
    "b200tfs_example_response_bound": (C.c_int, [C.c_int32, C.c_int32, _u64p, _u64p, _u64p]),
    "b200tfs_decode_example_responses": (C.c_int, [_vp, C.c_int32, _vp, C.c_int32, _u64p, _u64p, _vp, C.c_uint64, _vp, C.c_uint64]),
    "b200tfs_decode_example_responses_host_async": (C.c_int, [_vp, C.c_int32, _vp, C.c_int32, _u64p, _u64p, _vp, C.c_uint64, _vp,
                                                              C.c_uint64]),
    "b200tfs_example_response_results": (C.c_int, [_vp, C.c_int32, C.POINTER(C.c_int64), C.POINTER(ModelSpec), C.POINTER(C.c_int64)]),
    "b200tfs_example_tasks_request_size": (C.c_int, [C.POINTER(ExampleRequest), C.POINTER(ExampleTarget), C.POINTER(ExampleContext),
                                                     C.POINTER(ExampleTasks), _u64p]),
    "b200tfs_example_tasks_arena_size": (C.c_int, [C.c_int32, C.POINTER(ExampleRequest), C.POINTER(Bytes), C.POINTER(ExampleTarget),
                                                   C.POINTER(ExampleContext), C.POINTER(Bytes), C.POINTER(ExampleTasks), _u64p]),
    "b200tfs_encode_example_tasks_async": (C.c_int, [_vp, C.c_int32, C.POINTER(ExampleRequest), C.POINTER(Ragged), C.POINTER(Bytes),
                                                     C.POINTER(ExampleTarget), C.POINTER(ExampleContext), C.POINTER(Bytes),
                                                     C.POINTER(ExampleTasks), _vp, C.c_uint64]),
    "b200tfs_encode_example_tasks_host": (C.c_int, [_vp, C.c_int32, C.POINTER(ExampleRequest), C.POINTER(Ragged), C.POINTER(Bytes),
                                                    C.POINTER(ExampleTarget), C.POINTER(ExampleContext), C.POINTER(Bytes),
                                                    C.POINTER(ExampleTasks), _vp, C.c_uint64, _u64p, _u64p]),
    "b200tfs_example_sequences_request_size": (C.c_int, [C.POINTER(ExampleRequest), C.POINTER(ExampleTarget), C.POINTER(ExampleContext),
                                                         C.POINTER(ExampleTasks), C.POINTER(Ragged), C.POINTER(ExampleSequence), _u64p]),
    "b200tfs_example_sequences_arena_size": (C.c_int, [C.c_int32, C.POINTER(ExampleRequest), C.POINTER(Ragged), C.POINTER(Bytes),
                                                       C.POINTER(ExampleTarget), C.POINTER(ExampleContext), C.POINTER(Bytes),
                                                       C.POINTER(ExampleTasks), C.POINTER(ExampleSequence), _u64p]),
    "b200tfs_encode_example_sequences_async": (C.c_int, [_vp, C.c_int32, C.POINTER(ExampleRequest), C.POINTER(Ragged), C.POINTER(Bytes),
                                                         C.POINTER(ExampleTarget), C.POINTER(ExampleContext), C.POINTER(Bytes),
                                                         C.POINTER(ExampleTasks), C.POINTER(ExampleSequence), _vp, C.c_uint64]),
    "b200tfs_encode_example_sequences_host": (C.c_int, [_vp, C.c_int32, C.POINTER(ExampleRequest), C.POINTER(Ragged), C.POINTER(Bytes),
                                                        C.POINTER(ExampleTarget), C.POINTER(ExampleContext), C.POINTER(Bytes),
                                                        C.POINTER(ExampleTasks), C.POINTER(ExampleSequence), _vp, C.c_uint64, _u64p,
                                                        _u64p]),
    "b200tfs_example_specs_request_size": (C.c_int, [C.POINTER(ExampleRequest), C.POINTER(ExampleTarget), C.POINTER(ExampleContext),
                                                     C.POINTER(ExampleTasks), C.POINTER(Ragged), C.POINTER(ExampleSequence),
                                                     C.POINTER(RequestSpec), _u64p]),
    "b200tfs_example_specs_arena_size": (C.c_int, [C.c_int32, C.POINTER(ExampleRequest), C.POINTER(Ragged), C.POINTER(Bytes),
                                                   C.POINTER(ExampleTarget), C.POINTER(ExampleContext), C.POINTER(Bytes),
                                                   C.POINTER(ExampleTasks), C.POINTER(ExampleSequence), C.POINTER(RequestSpec), _u64p]),
    "b200tfs_encode_example_specs_async": (C.c_int, [_vp, C.c_int32, C.POINTER(ExampleRequest), C.POINTER(Ragged), C.POINTER(Bytes),
                                                     C.POINTER(ExampleTarget), C.POINTER(ExampleContext), C.POINTER(Bytes),
                                                     C.POINTER(ExampleTasks), C.POINTER(ExampleSequence), C.POINTER(RequestSpec), _vp,
                                                     C.c_uint64]),
    "b200tfs_encode_example_specs_host": (C.c_int, [_vp, C.c_int32, C.POINTER(ExampleRequest), C.POINTER(Ragged), C.POINTER(Bytes),
                                                    C.POINTER(ExampleTarget), C.POINTER(ExampleContext), C.POINTER(Bytes),
                                                    C.POINTER(ExampleTasks), C.POINTER(ExampleSequence), C.POINTER(RequestSpec), _vp,
                                                    C.c_uint64, _u64p, _u64p]),
    "b200tfs_example_lists_request_size": (C.c_int, [C.POINTER(ExampleRequest), C.POINTER(ExampleTarget), C.POINTER(ExampleContext),
                                                     C.POINTER(ExampleTasks), C.POINTER(Ragged), C.POINTER(ExampleSequence),
                                                     C.POINTER(RequestSpec), C.POINTER(ExampleLists), C.POINTER(Ragged), _u64p]),
    "b200tfs_example_lists_arena_size": (C.c_int, [C.c_int32, C.POINTER(ExampleRequest), C.POINTER(Ragged), C.POINTER(Bytes),
                                                   C.POINTER(ExampleTarget), C.POINTER(ExampleContext), C.POINTER(Bytes),
                                                   C.POINTER(ExampleTasks), C.POINTER(ExampleSequence), C.POINTER(RequestSpec),
                                                   C.POINTER(ExampleLists), C.POINTER(Ragged), C.POINTER(Bytes), _u64p]),
    "b200tfs_encode_example_lists_async": (C.c_int, [_vp, C.c_int32, C.POINTER(ExampleRequest), C.POINTER(Ragged), C.POINTER(Bytes),
                                                     C.POINTER(ExampleTarget), C.POINTER(ExampleContext), C.POINTER(Bytes),
                                                     C.POINTER(ExampleTasks), C.POINTER(ExampleSequence), C.POINTER(RequestSpec),
                                                     C.POINTER(ExampleLists), C.POINTER(Ragged), C.POINTER(Bytes), _vp, C.c_uint64]),
    "b200tfs_encode_example_lists_host": (C.c_int, [_vp, C.c_int32, C.POINTER(ExampleRequest), C.POINTER(Ragged), C.POINTER(Bytes),
                                                    C.POINTER(ExampleTarget), C.POINTER(ExampleContext), C.POINTER(Bytes),
                                                    C.POINTER(ExampleTasks), C.POINTER(ExampleSequence), C.POINTER(RequestSpec),
                                                    C.POINTER(ExampleLists), C.POINTER(Ragged), C.POINTER(Bytes), _vp, C.c_uint64, _u64p,
                                                    _u64p]),
    "b200tfs_example_device_lists_request_size": (C.c_int, [C.POINTER(ExampleRequest), C.POINTER(ExampleTarget),
                                                            C.POINTER(ExampleContext), C.POINTER(ExampleTasks), C.POINTER(Ragged),
                                                            C.POINTER(ExampleSequence), C.POINTER(RequestSpec), C.POINTER(ExampleLists),
                                                            C.POINTER(Ragged), C.POINTER(ExampleDeviceLists), _u64p]),
    "b200tfs_example_device_lists_arena_size": (C.c_int, [C.c_int32, C.POINTER(ExampleRequest), C.POINTER(Ragged), C.POINTER(Bytes),
                                                          C.POINTER(ExampleTarget), C.POINTER(ExampleContext), C.POINTER(Bytes),
                                                          C.POINTER(ExampleTasks), C.POINTER(ExampleSequence), C.POINTER(RequestSpec),
                                                          C.POINTER(ExampleLists), C.POINTER(Ragged), C.POINTER(Bytes),
                                                          C.POINTER(ExampleDeviceLists), _u64p]),
    "b200tfs_encode_example_device_lists_async": (C.c_int, [_vp, C.c_int32, C.POINTER(ExampleRequest), C.POINTER(Ragged),
                                                            C.POINTER(Bytes), C.POINTER(ExampleTarget), C.POINTER(ExampleContext),
                                                            C.POINTER(Bytes), C.POINTER(ExampleTasks), C.POINTER(ExampleSequence),
                                                            C.POINTER(RequestSpec), C.POINTER(ExampleLists), C.POINTER(Ragged),
                                                            C.POINTER(Bytes), C.POINTER(ExampleDeviceLists), _vp, C.c_uint64]),
    "b200tfs_encode_example_device_lists_host": (C.c_int, [_vp, C.c_int32, C.POINTER(ExampleRequest), C.POINTER(Ragged),
                                                           C.POINTER(Bytes), C.POINTER(ExampleTarget), C.POINTER(ExampleContext),
                                                           C.POINTER(Bytes), C.POINTER(ExampleTasks), C.POINTER(ExampleSequence),
                                                           C.POINTER(RequestSpec), C.POINTER(ExampleLists), C.POINTER(Ragged),
                                                           C.POINTER(Bytes), C.POINTER(ExampleDeviceLists), _vp, C.c_uint64, _u64p,
                                                           _u64p]),
    "b200tfs_multi_inference_response_bound": (C.c_int, [C.c_int32, _i32p, C.c_int32, _u64p, _u64p, _u64p]),
    "b200tfs_decode_multi_inference_responses": (C.c_int, [_vp, C.c_int32, _i32p, _vp, C.c_int32, _u64p, _u64p, _vpp, _u64p, _vpp,
                                                           _u64p]),
    "b200tfs_decode_multi_inference_responses_host_async": (C.c_int, [_vp, C.c_int32, _i32p, _vp, C.c_int32, _u64p, _u64p, _vpp,
                                                                      _u64p, _vpp, _u64p]),
    "b200tfs_multi_inference_response_results": (C.c_int, [_vp, C.c_int32, C.c_int32, C.POINTER(C.c_int64), C.POINTER(ModelSpec),
                                                           C.POINTER(C.c_int64)]),
}

_lib = None
_lib_lock = threading.Lock()


def load():
    """Load libb200tfs.so once and bind every declared symbol; RuntimeError if it is not built."""
    global _lib
    if _lib is not None:
        return _lib
    with _lib_lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is not built (run `python -c 'import __graft_entry__ as g; g.build()'` at the repo root); "
                "min_tfs_client has no CPU codec to fall back to"
            )
        lib = C.CDLL(LIB_PATH)
        for name, (restype, argtypes) in SIGNATURES.items():
            fn = getattr(lib, name)  # AttributeError = header/library out of sync: fail loudly
            fn.restype = restype
            fn.argtypes = argtypes
        _lib = lib
    return _lib


def last_error() -> str:
    return (load().b200tfs_last_error() or b"").decode("utf-8", "replace")


def check(code: int) -> None:
    """Map a status code to the exception the reference raises in the same situation."""
    if code == OK:
        return
    msg = last_error()
    if code in (E_DTYPE, E_SHAPE):
        raise ValueError(msg)
    if code == E_KEY:
        raise KeyError(msg)
    if code == E_RANGE:
        raise OverflowError(msg)
    if code == E_PARSE:
        from google.protobuf.message import DecodeError

        raise DecodeError(msg)
    if code == E_TOOBIG:
        raise ValueError(msg)
    if code == E_NONCANONICAL:
        raise NotImplementedError(msg)
    raise NativeError(code, msg)


def device_count() -> int:
    n = C.c_int32(0)
    rc = load().b200tfs_device_count(C.byref(n))
    return int(n.value) if rc == OK else 0


class PinnedBuffer:
    """Page-locked host memory exposed as a numpy uint8 array (``.array``)."""

    def __init__(self, nbytes: int):
        self.nbytes = int(nbytes)
        p = C.c_void_p()
        check(load().b200tfs_host_alloc(max(self.nbytes, 1), C.byref(p)))
        self.ptr = p.value
        self.array = np.ctypeslib.as_array((C.c_uint8 * max(self.nbytes, 1)).from_address(self.ptr))[: self.nbytes]

    def free(self):
        if self.ptr:
            self.array = None
            load().b200tfs_host_free(self.ptr)
            self.ptr = None

    def __del__(self):  # pragma: no cover - best effort
        try:
            self.free()
        except Exception:
            pass
