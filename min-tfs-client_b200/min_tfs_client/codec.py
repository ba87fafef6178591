"""GPU wire codec behind the drop-in API: numpy arrays <-> TensorProto / PredictRequest /
PredictResponse wire bytes, through ``libb200tfs.so`` (ctypes, no PyTorch).

What this replaces in the reference (paths relative to its checkout):
  encode  ``ndarray_to_tensor_proto`` + ``write_values_to_tensor_proto`` (tensors.py:17-35), the request
          assembly in ``_make_inference_request`` (requests.py:41-48) and ``SerializeToString``
          (prediction_service_pb2_grpc.py:52);
  decode  ``PredictResponse.FromString`` (…pb2_grpc.py:53), ``extract_shape`` and
          ``tensor_proto_to_ndarray`` (tensors.py:38-46).

A ``Codec`` owns one native context (one CUDA stream + scratch) and is not thread-safe; use
``get_codec()`` for a per-thread instance.  ``DT_STRING`` tensors are variable-length host objects:
their TensorProto is assembled on the host and spliced into the request by the kernel verbatim.
"""
from __future__ import annotations

import collections
import contextlib
import ctypes as C
import threading
from typing import Dict, Iterable, List, Mapping, Optional, Sequence, Tuple, Union

import numpy as np

from . import _native as N
from . import device as D
from .constants import BFLOAT16, DT_BFLOAT16, NP_TO_ENUM_MAPPING, enum_for_numpy, numpy_for_enum
from tensorflow.core.framework import types_pb2

DT_FLOAT, DT_HALF, DT_STRING = types_pb2.DT_FLOAT, types_pb2.DT_HALF, types_pb2.DT_STRING
DT_COMPLEX64, DT_COMPLEX128 = types_pb2.DT_COMPLEX64, types_pb2.DT_COMPLEX128

_ORDER = {"given": N.ORDER_GIVEN, "insertion": N.ORDER_GIVEN, "deterministic": N.ORDER_UPB, "upb": N.ORDER_UPB,
          "bytes": N.ORDER_BYTES}


def _as_enum(dtype) -> int:
    """DT_* enum from an enum int, a "DT_*" name or a numpy dtype."""
    if isinstance(dtype, (int, np.integer)):
        return int(dtype)
    if isinstance(dtype, str) and dtype.startswith("DT_"):
        return getattr(types_pb2, dtype)
    return enum_for_numpy(dtype)


def _validated_enum(arr) -> int:
    """Same gate as ``DataType(ndarray.dtype.type)`` (types.py:27-32): ValueError for foreign dtypes.  `arr`: anything with a numpy dtype."""
    t = arr.dtype.type
    if t in NP_TO_ENUM_MAPPING:
        return NP_TO_ENUM_MAPPING[t]
    if BFLOAT16 is not None and t is BFLOAT16:
        return DT_BFLOAT16
    allowed = ", ".join(k.__name__ for k in NP_TO_ENUM_MAPPING)
    raise ValueError(f"Dtype {t.__name__} is not valid. Allowable values: {allowed}")


def _string_tensor_proto_bytes(arr: np.ndarray) -> bytes:
    """Host assembly of a DT_STRING TensorProto (tensors.py:24, :10-14: str -> utf-8, bytes as is)."""
    from tensorflow.core.framework.tensor_pb2 import TensorProto
    from tensorflow.core.framework.tensor_shape_pb2 import TensorShapeProto

    proto = TensorProto(dtype=DT_STRING,
                        tensor_shape=TensorShapeProto(dim=[TensorShapeProto.Dim(size=d) for d in arr.shape]))
    proto.string_val.extend(v.encode("utf-8") if isinstance(v, str) else v for v in arr.ravel().tolist())
    return proto.SerializeToString()


def _bytes_tensor_proto_bytes(col: "BytesColumn") -> bytes:
    """Host assembly of the DT_STRING TensorProto of a host ``BytesColumn``: one string_val value of raw bytes per string."""
    from tensorflow.core.framework.tensor_pb2 import TensorProto
    from tensorflow.core.framework.tensor_shape_pb2 import TensorShapeProto

    proto = TensorProto(dtype=DT_STRING, tensor_shape=TensorShapeProto(dim=[TensorShapeProto.Dim(size=d) for d in col.shape]))
    o, d = col.offsets.tolist(), col.data
    proto.string_val.extend(d[o[j]: o[j + 1]].tobytes() for j in range(len(o) - 1))
    return proto.SerializeToString()


def _string_wire_dtype(key, wire_dtype) -> None:
    """ValueError when the wire dtype given for a string column is not DT_STRING."""
    if wire_dtype is not None and _as_enum(wire_dtype) != DT_STRING:
        raise ValueError(f"input {key!r}: a BytesColumn goes on the wire as DT_STRING, not {wire_dtype!r}")


def _check_host_offsets(key, col: "BytesColumn") -> None:
    """The offsets rule for host offsets, over the whole column: they never decrease and stay within ``0..data_len``."""
    if col.offsets_on_device:
        return
    o = col.offsets
    if o[0] < 0 or o[-1] > col.data_len or (o.size > 1 and (np.diff(o) < 0).any()):
        raise ValueError(f"input {key!r}: string offsets must rise within 0..{col.data_len}")


def _bytes_box(key, col: "BytesColumn", r0: int, row) -> "BytesColumn":
    """The strings of the box ``[r0 : r0 + row[0], :row[1], ...]`` of a padded host ``BytesColumn`` (``row``: a request's shape
    row, or its row count with every trailing dim full), in C order, as a column of their raw bytes.  Checks the offsets rule for
    the box alone - its first row's start, both ends of each of its strings, its last row's end never decrease and stay within
    ``0..data_len`` (ValueError) - as the device route does.  Work and memory are proportional to the box."""
    dims = col.shape
    bd = (int(row[0]),) + (tuple(int(x) for x in row[1:]) if len(row) > 1 else tuple(int(d) for d in dims[1:]))
    st = [int(np.prod(dims[a + 1:], dtype=np.int64)) for a in range(len(dims))]     # elements of one index of each axis
    idx = np.asarray(r0 * st[0], np.int64)
    for b, s in zip(bd, st):
        idx = idx[..., None] + np.arange(b, dtype=np.int64) * s
    flat = idx.ravel()
    o = col.offsets
    seq = np.concatenate([o[r0 * st[0]: r0 * st[0] + 1], np.stack([o[flat], o[flat + 1]], 1).ravel(),
                          o[(r0 + bd[0]) * st[0]: (r0 + bd[0]) * st[0] + 1]])
    if seq[0] < 0 or seq[-1] > col.data_len or (np.diff(seq) < 0).any():
        raise ValueError(f"input {key!r}: the string offsets of a request's box must rise within 0..{col.data_len}")
    lens = o[flat + 1] - o[flat]
    offsets = np.zeros(flat.size + 1, np.int64)
    np.cumsum(lens, out=offsets[1:])
    at = np.repeat(o[flat] - offsets[:-1], lens) + np.arange(int(offsets[-1]), dtype=np.int64)
    return BytesColumn(np.asarray(col.data)[at], offsets, bd)


class _PaddedString:
    """The Tensor struct of a string column of the padded encode (what the call reads of a _Prepared)."""

    __slots__ = ("key", "dims", "struct")

    def __init__(self, key: bytes, shape):
        self.key = key
        self.dims = (C.c_int64 * max(len(shape), 1))(*shape)
        self.struct = None


class _Prepared:
    """One input readied for the C ABI; keeps every buffer the Tensor struct points at alive."""

    __slots__ = ("array", "dims", "key", "struct", "on_device", "nbytes", "ndim", "size", "itemsize", "kind")

    def __init__(self, value, key: bytes, wire_dtype, tensor_content: bool, keep_snan: bool):
        if isinstance(value, BytesColumn):
            # raw strings, assembled on the host like a numpy str tensor (tensor_content / keep_snan do not apply to strings)
            if value.data_on_device or value.offsets_on_device:
                raise ValueError(f"input {key!r}: a BytesColumn of device arrays is encoded by encode_predict_requests_padded; "
                                 "encode_predict_requests takes host arrays")
            _string_wire_dtype(key, wire_dtype)
            _check_host_offsets(key, value)
            blob = np.frombuffer(_bytes_tensor_proto_bytes(value), dtype=np.uint8)
            self.on_device, self.array, self.dims, self.key = False, blob, (C.c_int64 * 1)(0), key
            self.struct = N.Tensor(data=blob.ctypes.data if blob.size else None, src_dtype=DT_STRING, wire_dtype=DT_STRING, rank=0,
                                   flags=N.F_PRESERIALIZED, dims=self.dims, key=key, key_len=len(key), packed_len=blob.size)
            self.nbytes, self.ndim, self.size, self.itemsize, self.kind = int(blob.size), 1, int(blob.size), 1, "u"
            return
        self.on_device = D.is_device_object(value)
        if self.on_device:
            # a tensor that already lives in HBM (CUDA array interface / DLPack): encoded in place, no host-to-device copy
            ptr, shape, dtype, keep = D.device_view(value)
            probe = np.empty(0, dtype=dtype)
            src_enum = _validated_enum(probe)
            if src_enum == DT_STRING or not dtype.isnative:
                raise ValueError("device inputs must be native-endian numeric arrays")
            wire_enum = src_enum if wire_dtype is None else _as_enum(wire_dtype)
            flags = N.F_DEVICE_DATA | (N.F_TENSOR_CONTENT if tensor_content else 0) | (N.F_KEEP_SNAN if keep_snan else 0)
            self.array = keep
            self.dims = (C.c_int64 * max(len(shape), 1))(*shape)
            n = int(np.prod(shape, dtype=np.int64))
            self.nbytes, self.ndim, self.size, self.itemsize, self.kind = n * dtype.itemsize, len(shape), n, dtype.itemsize, dtype.kind
            self.key = key
            self.struct = N.Tensor(data=ptr if n else None, src_dtype=src_enum, wire_dtype=wire_enum, rank=len(shape), flags=flags, dims=self.dims,
                                   key=key, key_len=len(key), packed_len=0)
            return
        arr = np.asarray(value)
        src_enum = _validated_enum(arr)
        flags = 0
        if src_enum == DT_STRING:
            blob = np.frombuffer(_string_tensor_proto_bytes(arr), dtype=np.uint8)
            self.array, self.dims = blob, (C.c_int64 * 1)(0)
            t = N.Tensor(data=blob.ctypes.data if blob.size else None, src_dtype=DT_STRING, wire_dtype=DT_STRING, rank=0,
                         flags=N.F_PRESERIALIZED, dims=self.dims, key=key, key_len=len(key), packed_len=blob.size)
        else:
            if not arr.dtype.isnative:
                arr = arr.astype(arr.dtype.newbyteorder("="))
            # C order, like ndarray.ravel() in tensors.py:34.  (np.ascontiguousarray promotes a 0-d array to shape (1,):
            # the reference keeps the empty shape - `tensor_shape {}` = 12 00 - so ask for the layout only.)
            arr = np.require(arr, requirements="C")
            wire_enum = src_enum if wire_dtype is None else _as_enum(wire_dtype)
            if tensor_content:
                flags |= N.F_TENSOR_CONTENT
            if keep_snan:
                flags |= N.F_KEEP_SNAN
            self.array = arr
            self.dims = (C.c_int64 * max(arr.ndim, 1))(*arr.shape)
            t = N.Tensor(data=arr.ctypes.data if arr.size else None, src_dtype=src_enum, wire_dtype=wire_enum, rank=arr.ndim,
                         flags=flags, dims=self.dims, key=key, key_len=len(key), packed_len=0)
        self.key = key
        self.struct = t
        a = self.array
        self.nbytes, self.ndim, self.size, self.itemsize, self.kind = int(a.nbytes), a.ndim, int(a.size), a.dtype.itemsize, a.dtype.kind


def _utf8(what: str, v) -> bytes:
    """A protobuf string field's bytes: ``str`` as UTF-8, ``bytes`` as given if they are valid UTF-8 (ValueError otherwise, as protobuf
    refuses them)."""
    if isinstance(v, str):
        return v.encode("utf-8")
    b = bytes(v)
    try:
        b.decode("utf-8")
    except UnicodeDecodeError:
        raise ValueError(f"{what} {b!r} is not valid UTF-8") from None
    return b


class _RequestSpec:
    """The signature_name, version_label and output_filter of one encode call as a ``b200tfs_request_spec`` (``struct``) and the
    bytes its fields point at; ``extra`` bounds the wire bytes they add to a request."""

    __slots__ = ("struct", "keep", "extra")

    def __init__(self, signature_name, version_label, output_filter):
        sig = b"" if signature_name is None else _utf8("signature_name", signature_name)
        label = None if version_label is None else _utf8("version_label", version_label)
        if isinstance(output_filter, (str, bytes)):
            raise TypeError("output_filter is a sequence of output names, not one name")
        names = [] if output_filter is None else [_utf8("output_filter name", x) for x in output_filter]
        ptrs = (C.c_char_p * max(len(names), 1))(*names)
        lens = (C.c_int64 * max(len(names), 1))(*[len(x) for x in names])
        self.struct = N.RequestSpec(signature_name=sig, signature_len=len(sig), version_label=label,
                                    version_label_len=-1 if label is None else len(label), output_filter=ptrs, output_filter_len=lens,
                                    n_output_filter=len(names))
        self.keep = (sig, label, names, ptrs, lens)
        self.extra = 32 + len(sig) + len(label or b"") + sum(11 + len(x) for x in names)

    @staticmethod
    def of(model_versions, signature_name=None, version_label=None, output_filter=None) -> Optional["_RequestSpec"]:
        """None when the call sets none of the three (its bytes are then those of a call without them)."""
        if signature_name is None and version_label is None and output_filter is None:
            return None
        if version_label is not None and any(v is not None for v in model_versions):
            raise ValueError("model_version and version_label are members of one oneof (ModelSpec.version_choice): give at most one")
        return _RequestSpec(signature_name, version_label, output_filter)

    @staticmethod
    def array(spec: Optional["_RequestSpec"], n: int):
        """n copies of the struct for the per-request _spec entry points (None: NULL)."""
        return None if spec is None else (N.RequestSpec * n)(*([spec.struct] * n))


def _wire_bound(p: "_Prepared", tensor_content: bool) -> int:
    """Upper bound of the bytes one prepared tensor occupies on the wire (payload + its own framing)."""
    frame = 64 + 16 * max(p.ndim, 1) + len(p.key)
    if p.struct.flags & N.F_PRESERIALIZED:
        return p.size + frame
    n = p.size
    if p.struct.src_dtype != p.struct.wire_dtype:
        return 4 * n + frame                      # f16 / bf16 -> DT_FLOAT
    if tensor_content or p.kind in "fc" and p.itemsize >= 4 or p.kind == "b":
        return p.nbytes + frame
    per = {1: 10, 2: 10, 4: 10, 8: 10} if p.kind == "i" else {1: 2, 2: 3, 4: 5, 8: 10}   # varint bytes per element
    return n * per[p.itemsize] + frame


_EXAMPLE_DTYPES = {np.dtype(t): _validated_enum(np.empty(0, t)) for t in (
    np.float16, np.float32, np.float64, np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint16, np.uint32, np.uint64, np.bool_)}


class BytesColumn:
    """A string tf.Example column (``bytes_list``) laid out as Arrow / cuDF hold one: a byte buffer ``data`` (``uint8[data_len]``)
    and ``offsets`` (``int[m + 1]``), string j being ``data[offsets[j]:offsets[j + 1]]``.  The m strings fill ``shape`` (default
    ``(m,)``) in C order: row i, ``shape[1:]`` strings, is example i's list; ``shape=()`` is one string repeated in every example,
    as a 0-d array is.  ``offsets[0]`` need not be 0 (a sliced column).

    Both may be numpy arrays (pageable or ``pinned_empty``; host offsets of any integer dtype) or device arrays
    (``__cuda_array_interface__`` / DLPack), so a GPU dataframe's string column is encoded where it lies; device offsets must be
    int64 (widen cuDF's int32 offsets first).  Each example's offsets must rise inside ``0..data_len``: host offsets are checked
    by the encode before anything runs, device ones by the kernels, and either way a request that breaks this raises ValueError.
    A ``RaggedColumn`` of a ``BytesColumn`` of shape ``[n, L, *inner]`` gives example i its first ``lengths[i]`` steps.
    ``from_array`` builds one from a numpy str / bytes array.
    """

    __slots__ = ("data", "offsets", "shape", "data_len", "data_on_device", "offsets_on_device")

    def __init__(self, data, offsets, shape=None):
        self.data_on_device = D.is_device_object(data)
        if self.data_on_device:
            _, dshape, ddtype, _ = D.device_view(data)
            if ddtype != np.uint8 or len(dshape) != 1:
                raise ValueError(f"string data must be a uint8 vector, got {ddtype} of shape {tuple(dshape)}")
            data_len = int(dshape[0])
        else:
            data = np.frombuffer(data, np.uint8) if isinstance(data, (bytes, bytearray, memoryview)) else np.asarray(data)
            if data.dtype != np.uint8 or data.ndim != 1:
                raise ValueError(f"string data must be a uint8 vector, got {data.dtype} of shape {data.shape}")
            data = np.require(data, requirements="C")
            data_len = data.size
        self.offsets_on_device = D.is_device_object(offsets)
        if self.offsets_on_device:
            _, oshape, odtype, _ = D.device_view(offsets)
            if odtype != np.int64:
                raise ValueError(f"device string offsets must be int64, got {odtype} (cast cuDF's int32 offsets to int64 first)")
            oshape = tuple(oshape)
        else:
            offsets = np.asarray(offsets)
            if offsets.dtype.kind not in "iu":
                raise ValueError(f"string offsets must be integers, got {offsets.dtype}")
            if offsets.dtype == np.uint64 and offsets.size and offsets.max() > np.iinfo(np.int64).max:
                raise ValueError("string offsets exceed int64")
            offsets = np.require(offsets.astype(np.int64, copy=False), requirements="CA")
            oshape = offsets.shape
        if len(oshape) != 1 or oshape[0] < 1:
            raise ValueError(f"string offsets are a vector of at least one entry, got shape {oshape}")
        shape = (oshape[0] - 1,) if shape is None else tuple(int(x) for x in shape)
        if int(np.prod(shape, dtype=np.int64)) != oshape[0] - 1:
            raise ValueError(f"{oshape[0] - 1} strings do not fill shape {shape}")
        self.data, self.offsets, self.shape, self.data_len = data, offsets, shape, data_len

    @classmethod
    def from_array(cls, a) -> "BytesColumn":
        """The strings of a numpy str (``U``) or bytes (``S``) array, as ``examples_from_input_dict`` makes them: trailing NULs
        dropped (inner ones kept), str encoded as UTF-8 (a lone surrogate raises ``UnicodeEncodeError``)."""
        a = np.asarray(a)
        if a.dtype.kind == "U":
            enc = np.asarray(np.char.encode(a, "utf-8"))
        elif a.dtype.kind == "S":
            enc = a
        else:
            raise ValueError(f"BytesColumn.from_array takes str or bytes arrays, got {a.dtype}")
        m, w = enc.size, enc.dtype.itemsize
        cells = np.ascontiguousarray(enc).reshape(m).view(np.uint8).reshape(m, w)
        nz = cells != 0
        lens = np.where(nz.any(axis=1), w - np.argmax(nz[:, ::-1], axis=1), 0) if w else np.zeros(m, np.int64)
        data = cells[np.arange(w) < lens[:, None]]
        offsets = np.zeros(m + 1, np.int64)
        np.cumsum(lens, out=offsets[1:])
        return cls(data, offsets, a.shape)

    @property
    def ndim(self) -> int:
        return len(self.shape)

    def strings(self, i: int, count: Optional[int] = None) -> List[bytes]:
        """The first ``count`` (default: all) strings of example i (host arrays)."""
        row = int(np.prod(self.shape[1:], dtype=np.int64)) if self.shape else 1
        base = i * row if self.shape else 0
        o = np.asarray(self.offsets)[base: base + (row if count is None else count) + 1].tolist()
        d = np.asarray(self.data)
        return [d[o[j]: o[j + 1]].tobytes() for j in range(len(o) - 1)]

    def _bind(self, keep: list, upload=None):
        """(data pointer, or None when ``data_len`` is 0; the ``N.Bytes`` entry of the offsets) for the C ABI.  Every array the two
        point at is appended to ``keep``.  With ``upload`` (a Codec), host arrays are first copied to its device."""
        def ptr(a, on_device, dtype):
            if on_device:
                p, _, _, hold = D.device_view(a)
            elif upload is not None:
                hold = upload.device_array(np.ascontiguousarray(a, dtype=dtype))
                p = hold.ptr
            else:
                hold, p = a, a.ctypes.data
            keep.append(hold)
            return p

        data = ptr(self.data, self.data_on_device, np.uint8) if self.data_len else None
        offsets = ptr(self.offsets, self.offsets_on_device, np.int64)
        flags = N.F_DEVICE_DATA if self.offsets_on_device or upload is not None else 0
        return data, N.Bytes(offsets=offsets, data_len=self.data_len, flags=flags)


class RaggedColumn:
    """A variable-length tf.Example column - what a model parses as ``VarLenFeature`` / ``RaggedFeature``: a click history, the
    token ids of a query, multi-hot ids.  Example i's feature holds ``values[i, :lengths[i]].ravel()``, converted as a dense row is.

    ``values`` has shape ``[n, L, *inner]`` (rank >= 2): a numpy array (pageable or ``pinned_empty``), a device array
    (``__cuda_array_interface__`` / DLPack) or a ``BytesColumn`` of that shape.  ``lengths`` is ``int[n]``: a numpy array of any
    integer dtype, whose values must lie in ``0..L`` (ValueError here), or a device array of int64, whose values the encode kernels
    check (ValueError from the encode).
    """

    __slots__ = ("values", "lengths", "shape", "lengths_on_device")

    def __init__(self, values, lengths):
        shape = values.shape if isinstance(values, BytesColumn) else \
            tuple(D.device_view(values)[1]) if D.is_device_object(values) else np.shape(values)
        if len(shape) < 2:
            raise ValueError(f"ragged values have shape [n, L, *inner] (rank >= 2), got {shape}")
        self.lengths_on_device = D.is_device_object(lengths)
        if self.lengths_on_device:
            _, lshape, ldtype, _ = D.device_view(lengths)
            if ldtype != np.int64:
                raise ValueError(f"device ragged lengths must be int64, got {ldtype}")
        else:
            lengths = np.asarray(lengths)
            if lengths.dtype.kind not in "iu":
                raise ValueError(f"ragged lengths must be integers, got {lengths.dtype}")
            lshape = lengths.shape
        if tuple(lshape) != shape[:1]:
            raise ValueError(f"ragged lengths of shape {tuple(lshape)} for values of {shape[0]} examples")
        if not self.lengths_on_device:
            if ((lengths < 0) | (lengths > shape[1])).any():
                raise ValueError(f"ragged lengths must lie in 0..{shape[1]}")
            lengths = np.ascontiguousarray(lengths, dtype=np.int64)
        self.values, self.lengths, self.shape = values, lengths, shape

    @property
    def ndim(self) -> int:
        return len(self.shape)

    def row(self, i: int) -> np.ndarray:
        """Example i's values, ``[lengths[i], *inner]`` (host arrays)."""
        return np.asarray(self.values)[i, :int(self.lengths[i])]

    def strings(self, i: int) -> List[bytes]:
        """Example i's strings, when the values are a ``BytesColumn`` (host arrays)."""
        return self.values.strings(i, int(self.lengths[i]) * int(np.prod(self.shape[2:], dtype=np.int64)))


class _ExampleColumn(tuple):
    """(Feature, keep-alive, key, Ragged or None), and ``bytes_entry``: the Bytes entry of a string column (None otherwise)."""

    bytes_entry = None


def _example_columns(input_dict: Mapping, context: bool = False):
    """(n_examples, [_ExampleColumn (Feature, keep-alive, key, Ragged or None), ...]) for the device route, or None for a request
    ``examples_from_input_dict`` assembles on the host (numpy str / bytes columns, dtypes without a device conversion - which it
    rejects or converts itself).  A ``RaggedColumn`` gives the Feature of its padded ``values`` (``row_elems = L * unit``) and a
    Ragged entry for its lengths; a ``BytesColumn`` a DT_STRING Feature of its byte buffer and a Bytes entry for its offsets.
    Raises the ValueError ``examples_from_input_dict`` raises for disagreeing example counts, and for device arrays of a dtype the
    device route does not take.  With ``context``, ``input_dict`` is a context: every value is one row of all its values (a
    ``RaggedColumn`` raises ValueError, as ``examples_with_context_from_input_dict`` does)."""
    cols = []
    for k, v in input_dict.items():
        key = k.encode("utf-8") if isinstance(k, str) else bytes(k)
        rag = v if isinstance(v, RaggedColumn) else None
        if rag is not None:
            if context:
                raise ValueError(f"context {k!r}: a RaggedColumn has no place in a context, which has no example axis")
            v = rag.values
        if isinstance(v, BytesColumn):
            cols.append((key, None, v.shape, None, v, v.data_on_device, rag))
        elif D.is_device_object(v):
            ptr, shape, dtype, hold = D.device_view(v)
            if dtype not in _EXAMPLE_DTYPES:
                raise ValueError(f"input {k!r}: device arrays of dtype {dtype} have no tf.Example feature kind on the device")
            cols.append((key, ptr, shape, dtype, hold, True, rag))
        else:
            a = np.asarray(v)
            dtype = a.dtype.newbyteorder("=")
            if dtype not in _EXAMPLE_DTYPES:
                return None
            cols.append((key, None, a.shape, dtype, a, False, rag))
    if context:     # one example, whose row is the whole value
        cols = [(c[0], c[1], (1, int(np.prod(c[2], dtype=np.int64))), *c[3:]) for c in cols]
    rows = {shape[0] for _, _, shape, _, _, _, _ in cols if len(shape)}
    if len(rows) > 1:
        raise ValueError(f"inputs disagree on the number of examples: {sorted(rows)}")
    n = rows.pop() if rows else (1 if cols else 0)
    preps = []
    for key, ptr, shape, dtype, hold, on_device, rag in cols:
        row_elems = int(np.prod(shape[1:], dtype=np.int64)) if len(shape) else 1
        flags = 0 if len(shape) else N.F_BROADCAST
        if on_device:
            flags |= N.F_DEVICE_DATA
        b = None
        if isinstance(hold, BytesColumn):
            col, hold = hold, []
            ptr, b = col._bind(hold)
            f = N.Feature(data=ptr, src_dtype=DT_STRING, flags=flags, row_elems=row_elems, key=key, key_len=len(key))
        else:
            if not on_device:
                hold = np.require(hold.astype(dtype, copy=False), requirements="CA")
                ptr = hold.ctypes.data
            size = int(np.prod(shape, dtype=np.int64))
            f = N.Feature(data=ptr if size else None, src_dtype=_EXAMPLE_DTYPES[dtype], flags=flags, row_elems=row_elems,
                          key=key, key_len=len(key))
        g = None
        if rag is not None:
            if rag.lengths_on_device:
                lptr, _, _, lhold = D.device_view(rag.lengths)
            else:
                lhold = rag.lengths
                lptr = lhold.ctypes.data
            g = N.Ragged(lengths=lptr or None, max_len=shape[1], unit=int(np.prod(shape[2:], dtype=np.int64)),
                         flags=N.F_DEVICE_DATA if rag.lengths_on_device else 0)
            hold = (hold, lhold)
        col = _ExampleColumn((f, hold, key, g))
        col.bytes_entry = b
        preps.append(col)
    return n, preps


def _head_rows(v, n: int):
    """The first n rows of an input value (0-d values as they are), for a request the host assembles."""
    if isinstance(v, RaggedColumn):
        return RaggedColumn(_head_rows(v.values, n), v.lengths[:n])
    if isinstance(v, BytesColumn):
        per = int(np.prod(v.shape[1:], dtype=np.int64)) if len(v.shape) else 0
        return BytesColumn(v.data, v.offsets[:n * per + 1], (n, *v.shape[1:])) if len(v.shape) else v
    a = np.asarray(v)
    return a[:n] if a.ndim else a


def _shape_of(v) -> Tuple[int, ...]:
    if isinstance(v, (BytesColumn, RaggedColumn)):
        return tuple(v.shape)
    return tuple(D.device_view(v)[1]) if D.is_device_object(v) else tuple(np.shape(v))


def _sequence_count(context_dict: Mapping, feature_list_dict: Mapping) -> int:
    """The number of SequenceExamples ``context_dict`` and ``feature_list_dict`` hold: the leading dimension of every non-0-d
    context value and every feature-list value (ValueError when they disagree, or for a feature-list value of rank < 2, which
    has no step axis); with no such value 1 when either dict is non-empty, else 0."""
    rows = set()
    for k, v in feature_list_dict.items():
        shape = _shape_of(v)
        if len(shape) < 2:
            raise ValueError(f"feature list {k!r}: values have shape [n, T, *inner] (rank >= 2), got {shape}")
        rows.add(shape[0])
    rows |= {s[0] for s in map(_shape_of, context_dict.values()) if len(s)}
    if len(rows) > 1:
        raise ValueError(f"inputs disagree on the number of sequences: {sorted(rows)}")
    return rows.pop() if rows else (1 if context_dict or feature_list_dict else 0)


def _host_example_request(model_name, model_version, input_dict, grpc_frame: bool, predict_input=None, context_dict=None,
                          tasks=None, **fields) -> bytes:
    """A request with a column the device route does not take, as ``examples_from_input_dict`` and protobuf make it: a
    ClassificationRequest, or with ``predict_input`` a PredictRequest whose input of that key is the DT_STRING ``[n]`` tensor of
    the examples, each serialized with ``deterministic=True``.  With ``context_dict`` the examples and the context form an
    ExampleListWithContext (``examples_with_context_from_input_dict``): the ClassificationRequest's input, or the one string of a
    DT_STRING ``[1]`` tensor.  With ``tasks`` the request is the MultiInferenceRequest ``make_multi_inference_request`` builds.
    ``fields``: signature_name / version_label / output_filter (``requests.apply_spec_fields``)."""
    from .requests import (TensorServingClient, apply_spec_fields, examples_from_input_dict, examples_with_context_from_input_dict,
                           make_multi_inference_request)

    if tasks is not None:
        req = make_multi_inference_request(model_name, model_version, tasks, input_dict, context_dict)
    elif predict_input is None:
        from tensorflow_serving.apis.classification_pb2 import ClassificationRequest

        req = TensorServingClient._make_example_request(None, ClassificationRequest, model_name, input_dict, model_version, context_dict)
    else:
        from tensorflow_serving.apis.predict_pb2 import PredictRequest

        req = PredictRequest()
        req.model_spec.name = model_name
        if model_version is not None:
            req.model_spec.version.value = model_version
        if context_dict is None:
            values = examples_from_input_dict(input_dict).example_list.examples
        else:
            values = [examples_with_context_from_input_dict(input_dict, context_dict).example_list_with_context]
        key = predict_input.decode("utf-8") if isinstance(predict_input, bytes) else predict_input
        t = req.inputs[key]
        t.dtype = DT_STRING
        t.tensor_shape.dim.add().size = len(values)
        t.string_val.extend(e.SerializeToString(deterministic=True) for e in values)
    wire = apply_spec_fields(req, model_version, **fields).SerializeToString(deterministic=True)
    return (b"\x00" + len(wire).to_bytes(4, "big") + wire) if grpc_frame else wire


class DecodedSpec:
    """model_spec of a parsed response (model.proto:9-33)."""

    __slots__ = ("name", "version", "has_version", "version_label", "signature_name")

    def __init__(self, name="", version=0, has_version=False, version_label="", signature_name=""):
        self.name, self.version, self.has_version = name, version, has_version
        self.version_label, self.signature_name = version_label, signature_name

    def __repr__(self):
        return (f"DecodedSpec(name={self.name!r}, version={self.version}, has_version={self.has_version}, "
                f"version_label={self.version_label!r}, signature_name={self.signature_name!r})")


_FUSED_MOVES = frozenset((1, 2, 8, 18))   # DT_FLOAT, DT_DOUBLE, DT_COMPLEX64, DT_COMPLEX128: what decode_fused_kernel moves itself
# the dtypes whose values are packed varints (int_val, int64_val, uint32_val, uint64_val, bool_val, half_val): what the same launch
# decodes as well once b200tfs_set_decode_varints is on
_VARINT_DTYPES = frozenset((3, 4, 5, 6, 9, 10, 14, 17, 19, 22, 23))


def _narrowing_cast(out_dtypes: Mapping) -> Optional[int]:
    """DT_HALF or DT_BFLOAT16 when every requested cast is that one narrowing of float32 (b200tfs_set_decode_cast does it in
    the decode launch itself), else None."""
    try:
        wanted = {int(enum_for_numpy(np.dtype(v).type)) for v in out_dtypes.values()}
    except (KeyError, ValueError, TypeError):
        return None
    if len(wanted) == 1 and next(iter(wanted)) in (int(DT_HALF), int(DT_BFLOAT16)):
        return next(iter(wanted))
    return None


def _narrowing_fits(dtype: int, key, out_dtypes: Mapping) -> bool:
    """The narrowing cast applies to every float32 output: it is right only when exactly those were asked for."""
    return (int(dtype) == DT_FLOAT) == (key in out_dtypes)


def _to_unpack(o: N.Output, unfinished: int = N.E_SIZE) -> bool:
    """Make a table entry a device decode did not finish - a varint output it decoded with an error, or status `unfinished`
    (E_SIZE: no room in the fused launch's slot) - read as the walk tabulated it: status OK, no OF_DEVICE_VARINT.  The unpack
    route then finishes it and raises what it raises for it.  False for an entry with an error of its own."""
    if not (o.flags & N.OF_DEVICE_VARINT or o.status in (N.OK, unfinished)):
        return False
    o.flags &= ~N.OF_DEVICE_VARINT
    o.status = N.OK
    return True


def _stored(o: N.Output) -> bool:
    """Whether the fused launch stored this output in its slot: a dtype it moves itself, or a varint output it decoded.  Decided
    before _resolve_output, which may raise.  An output the launch did not finish goes to the unpack route."""
    if o.flags & N.OF_DEVICE_VARINT and o.status == N.OK:
        return True
    if o.flags & N.OF_DEVICE_VARINT or o.status == N.E_SIZE:
        _to_unpack(o)
        return False
    return o.status == N.OK and int(o.dtype) in _FUSED_MOVES and bool(o.n_runs and o.n_elems)


def _stored_as(o: N.Output, dst_code: int, cast_code: int = 0) -> bool:
    """Whether the resolved destination dtype is what the launch wrote: the output's own, or the narrowing of a float32 output
    (strict DT_HALF resolves to half_val read as values, the launch wrote TF's bit patterns)."""
    return dst_code == int(o.dtype) or bool(cast_code) and int(o.dtype) == DT_FLOAT and dst_code == cast_code


def _check_out(key, dst, dtype, shape, contiguous: bool = False):
    """ValueError unless the caller's destination `dst` (``out={key: dst}``) holds exactly `dtype` and `shape` - and, with
    `contiguous`, a numpy one is C-contiguous.  Returns (pointer, keep-alive) of a device destination, None for a numpy one."""
    shape = tuple(shape)
    if D.is_device_object(dst):
        ptr, dshape, ddtype, keep = D.device_view(dst)
        if ddtype != dtype or tuple(dshape) != shape:
            raise ValueError(f"out[{key!r}]: {ddtype}{tuple(dshape)} does not match the decoded {dtype}{shape}")
        return ptr, keep
    if not isinstance(dst, np.ndarray) or dst.dtype != dtype or dst.shape != shape or (contiguous and not dst.flags.c_contiguous):
        raise ValueError(f"out[{key!r}] does not match the decoded {dtype}{shape}")
    return None


# what one fused launch left on the host: n records staged in buf at off, their outputs in dst (a slot of stride bytes per
# record), each record's table ({key: Output}) and model_spec
_Launch = collections.namedtuple("_Launch", "n buf off dst stride tables specs")

# what a per-key device decode (Codec._key_device) left: its key structs, the wire on the device, the results table, each
# response's status and DecodedSpec, and the destinations as Codec._key_deliver takes them (holds: their keep-alives)
_KeyLaunch = collections.namedtuple("_KeyLaunch", "keys wire outs rec_status specs shapes np_types dev ptrs holds")

# one response's DT_STRING output as the runtime gives it: string_val's raw bytes and the shape (-1 inferred)
_RawStrings = collections.namedtuple("_RawStrings", "strings shape")


class OpenResponse:
    """One PredictResponse after the fused launch: the table, and the host buffer the fixed-width outputs landed in."""

    def __init__(self, codec, buf, base, dst, table):
        self._codec, self._buf, self._base, self._dst, self.table = codec, buf, base, dst, table
        self._stored = {k for k, o in table.items() if _stored(o)}
        self._handed = set()

    def wire_of(self, key) -> bytes:
        o = self.table[key]
        return self._buf[self._base + o.msg_off: self._base + o.msg_off + o.msg_len].tobytes()

    def array(self, key, strict: bool) -> Optional[np.ndarray]:
        """The decoded output, or None when the launch did not move it (varint-packed, string, tensor_content only): the
        caller then decodes ``wire_of(key)`` on its own.  Raises what the reference raises for this output."""
        o = self.table[key]
        if key not in self._stored:
            return None
        np_type, dst_code, shape = self._codec._resolve_output(o, strict, None)
        if not _stored_as(o, dst_code):
            return None
        at = int(o.dst_off)
        arr = self._dst[at: at + int(o.dst_bytes)].view(np_type).reshape(shape)
        if key in self._handed:      # tensor_proto_to_ndarray returns a fresh array per call (tensors.py:46): never alias two results
            return arr.copy()
        self._handed.add(key)
        return arr


class RegressionBatch:
    """A batch of RegressionResponses decoded into one array: ``values`` float32 ``[rows]`` (response 0's regressions, then
    response 1's, ...), ``counts`` int64 ``[n]`` (regressions per response), ``specs`` (a ``DecodedSpec`` per response)."""

    __slots__ = ("values", "counts", "specs")

    def __init__(self, values, counts, specs):
        self.values, self.counts, self.specs = values, counts, specs


class ClassificationBatch:
    """A batch of ClassificationResponses decoded into one array: ``scores`` float32 ``[rows, C]``, ``counts`` int64 ``[n]``,
    ``specs``; ``class_labels`` is the list of the C labels when every example lists the same labels in the same order (else
    None), and ``labels()`` gives every example's labels."""

    __slots__ = ("scores", "counts", "specs", "class_labels", "_rows")

    def __init__(self, scores, counts, specs, class_labels, rows):
        self.scores, self.counts, self.specs, self.class_labels, self._rows = scores, counts, specs, class_labels, rows

    def labels(self) -> List[List[str]]:
        """Per example, the labels of its classes (a callable: the common case decodes only C strings)."""
        rows = self._rows
        if callable(rows):
            rows = self._rows = rows()
        return [list(r) for r in rows]


class ParsedResponse:
    """Table the parse kernel produced for one PredictResponse: where every output's values lie."""

    def __init__(self, wire, offset: int, length: int, status: int, outputs: Dict[str, N.Output], spec: DecodedSpec):
        self.wire, self.offset, self.length = wire, offset, length
        self.status, self.outputs, self.model_spec = status, outputs, spec

    def keys(self):
        return self.outputs.keys()


class Codec:
    def __init__(self, device: int = 0):
        self._lib = N.load()
        ctx = C.c_void_p()
        rc = self._lib.b200tfs_create(device, C.byref(ctx))
        if rc != N.OK:
            raise RuntimeError(f"cannot create a GPU codec context on device {device}: {N.last_error()}")
        self._ctx = ctx
        self.device = device
        self._pinned = D.PinnedArrays()
        self._wire_pinned = None      # page-locked landing buffer of encode(..., out="pinned")
        # whether a response decoded so far carried packed-varint outputs.  Until then the single-launch decode leaves them to the
        # unpack route and float-only traffic pays nothing; from then on every call sizes its slots from its own records
        # (_slot_stride) and the launch decodes varint outputs too when they have some (b200tfs_set_decode_varints)
        self._seen_varints = False
        # decode_predict_responses_concat calls the device route finished (the others were decoded response by response)
        self.concat_device_calls = 0
        # decode_predict_responses_padded calls the device route finished
        self.padded_device_calls = 0
        # encode_predict_requests_padded calls the device route finished
        self.padded_encode_device_calls = 0
        self._pe_arena = None         # their device arena (grows)
        # decode_regression_responses / decode_classification_responses calls the device route finished
        self.example_response_device_calls = 0
        self.multi_inference_device_calls = 0     # MultiInference batches the device route decoded
        self._xr_scratch = None       # their device destinations when the result goes to host memory: (values, labels)

    def close(self):
        if getattr(self, "_ctx", None):
            if self._pe_arena is not None:
                self._pe_arena.free()
                self._pe_arena = None
            self._lib.b200tfs_destroy(self._ctx)
            self._ctx = None
            self._pinned.release()
            if self._wire_pinned is not None:
                self._wire_pinned.free()
                self._wire_pinned = None

    # ---- page-locked and device-resident arrays ---------------------------------------------------
    def pinned_empty(self, shape, dtype=np.float32) -> np.ndarray:
        """An uninitialised page-locked numpy array (lives until the codec is closed).  Inputs that sit in one are copied by the
        DMA engines at the PCIe rate; handed to ``decode_predict_response(..., out={key: arr})`` the decoded tensor lands in it
        directly."""
        return self._pinned.empty(shape, dtype)

    def device_array(self, array) -> "D.DeviceArray":
        """Upload `array` once; the returned device array can be encoded any number of times without a host-to-device copy."""
        a = np.require(np.asarray(array), requirements="C")
        return D.DeviceArray(self, a.shape, a.dtype).copy_from_host(a)

    def _pinned_wire(self, cap: int) -> "N.PinnedBuffer":
        if self._wire_pinned is None or self._wire_pinned.nbytes < cap:
            if self._wire_pinned is not None:
                self._wire_pinned.free()
            self._wire_pinned = N.PinnedBuffer(max(cap, 1 << 20))
        return self._wire_pinned

    def __del__(self):  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass

    # ---- plumbing -----------------------------------------------------------------------------
    @property
    def ctx(self):
        return self._ctx

    def sync(self):
        N.check(self._lib.b200tfs_sync(self._ctx))

    def kernel_launches(self) -> int:
        n = C.c_uint64(0)
        N.check(self._lib.b200tfs_kernel_launches(self._ctx, C.byref(n)))
        return int(n.value)

    # ---- encode --------------------------------------------------------------------------------
    def encode_tensor_protos(self, arrays: Sequence, *, wire_dtype=None, tensor_content: bool = False,
                             keep_snan: bool = False) -> List[bytes]:
        """Wire bytes of ``ndarray_to_tensor_proto(a).SerializeToString()`` for each array."""
        preps = [_Prepared(a, b"", wire_dtype, tensor_content, keep_snan) for a in arrays]
        n = len(preps)
        if n == 0:
            return []
        out: List[Optional[bytes]] = [None] * n
        dev_idx = []
        for i, p in enumerate(preps):  # a bare DT_STRING proto is host bytes already
            if p.struct.flags & N.F_PRESERIALIZED:
                out[i] = p.array.tobytes()
            else:
                dev_idx.append(i)
        if dev_idx:
            ts = (N.Tensor * len(dev_idx))(*[preps[i].struct for i in dev_idx])
            cap = sum(_wire_bound(preps[i], tensor_content) + 512 for i in dev_idx)
            wire = np.empty(cap, dtype=np.uint8)
            off = (C.c_uint64 * len(dev_idx))()
            ln = (C.c_uint64 * len(dev_idx))()
            N.check(self._lib.b200tfs_encode_tensor_protos_host(self._ctx, len(dev_idx), ts, wire.ctypes.data, cap, off, ln))
            for j, i in enumerate(dev_idx):
                out[i] = wire[off[j]: off[j] + ln[j]].tobytes()
        return out  # type: ignore[return-value]

    def _build_requests(self, requests, order, wire_dtype, tensor_content, keep_snan, grpc_frame=False):
        order_code = _ORDER[order] if isinstance(order, str) else int(order)
        keep = []
        structs = []
        for model_name, model_version, inputs in requests:
            items = list(inputs.items()) if isinstance(inputs, Mapping) else list(inputs)
            preps = []
            for k, v in items:
                kb = k.encode("utf-8") if isinstance(k, str) else bytes(k)
                wd = wire_dtype.get(k) if isinstance(wire_dtype, Mapping) else wire_dtype
                preps.append(_Prepared(v, kb, wd, tensor_content, keep_snan))
            arr = (N.Tensor * max(len(preps), 1))(*[p.struct for p in preps])
            name = model_name.encode("utf-8") if isinstance(model_name, str) else bytes(model_name)
            req = N.Request(model_name=name, model_name_len=len(name), has_version=int(model_version is not None), order=order_code,
                            version=int(model_version) if model_version is not None else 0, n_inputs=len(preps), flags=N.RF_GRPC_FRAME if grpc_frame else 0,
                            inputs=arr)
            keep.append((preps, arr, name))
            structs.append(req)
        return keep, structs

    def encode_predict_requests(self, requests: Iterable[Tuple[str, Optional[int], Union[Mapping, Sequence]]], *,
                                order="deterministic", wire_dtype=None, tensor_content: bool = False,
                                keep_snan: bool = False, grpc_frame: bool = False, out=None, signature_name=None,
                                version_label=None, output_filter=None) -> List[bytes]:
        """Each item is ``(model_name, model_version, inputs)``; returns one PredictRequest wire per item.

        The bytes equal ``PredictRequest.SerializeToString(deterministic=True)`` of the message the
        reference builds in requests.py:41-48 (``order="deterministic"``), or list the map entries in
        the order given (``order="given"``).  ``grpc_frame=True`` puts gRPC's five-byte length-prefixed-message
        header in front (for a transport that writes HTTP/2 DATA frames itself; grpc-python adds it on its own).
        Inputs may be numpy arrays (pageable or ``pinned_empty``) or device arrays (``__cuda_array_interface__`` / DLPack: no
        host-to-device copy).  ``out="pinned"`` returns uint8 views of the codec's page-locked landing buffer instead of ``bytes``
        objects (no copy on the host; valid until the next encode on this codec).  A DT_STRING input may be a numpy str array
        (UTF-8, as the reference) or a ``BytesColumn`` of host arrays: a DT_STRING tensor of its shape whose ``string_val`` holds
        each string's raw bytes (NULs and high bytes kept), so binary data such as an encoded image can be sent; its offsets must
        rise within ``0..data_len`` and ``wire_dtype`` must be DT_STRING if given (ValueError).  A ``BytesColumn`` of device arrays
        raises ValueError: ``encode_predict_requests_padded`` encodes those on the device.

        ``signature_name``, ``version_label`` and ``output_filter`` (a sequence of output names) set ``model_spec.signature_name``,
        ``model_spec.version_label`` and ``output_filter`` of every request of the call (``str``, or ``bytes`` that are valid UTF-8).
        ``version_label`` is in a oneof with the version: a request with a ``model_version`` raises ValueError.  None leaves a field
        unset, and the bytes are those of a call without it.
        """
        requests = list(requests)
        spec = _RequestSpec.of([v for _, v, _ in requests], signature_name, version_label, output_filter)
        keep, structs = self._build_requests(requests, order, wire_dtype, tensor_content, keep_snan, grpc_frame)
        n = len(structs)
        if n == 0:
            return []
        reqs = (N.Request * n)(*structs)
        specs = _RequestSpec.array(spec, n)
        if out is not None and out != "pinned":
            raise ValueError('out must be None or "pinned"')
        if n == 1 and out is None:
            # one request whose size is closed-form (no varint-packed input): copy straight into the bytes object
            total = C.c_uint64()
            if _HAVE_NEW_BYTES and self._lib.b200tfs_request_size_spec(reqs, specs, C.byref(total)) == N.OK:
                obj, addr = _new_bytes(int(total.value))
                off = (C.c_uint64 * 1)()
                ln = (C.c_uint64 * 1)()
                N.check(self._lib.b200tfs_encode_requests_host_spec(self._ctx, 1, reqs, specs, addr, total.value, off, ln))
                if off[0] != 0 or ln[0] != total.value:
                    raise N.NativeError(N.E_ARG, f"encoded length {ln[0]} at {off[0]} does not match the planned {total.value}")
                return [obj]
        cap = 0
        for preps, _, name in keep:
            cap += 1024 + len(name) + (spec.extra if spec else 0)
            for p in preps:
                cap += _wire_bound(p, tensor_content) + 512
        off = (C.c_uint64 * n)()
        ln = (C.c_uint64 * n)()
        if out == "pinned":
            pw = self._pinned_wire(cap)
            N.check(self._lib.b200tfs_encode_requests_host_spec(self._ctx, n, reqs, specs, pw.ptr, cap, off, ln))
            return [pw.array[off[i]: off[i] + ln[i]] for i in range(n)]
        wire = np.empty(cap, dtype=np.uint8)
        N.check(self._lib.b200tfs_encode_requests_host_spec(self._ctx, n, reqs, specs, wire.ctypes.data, cap, off, ln))
        return [wire[off[i]: off[i] + ln[i]].tobytes() for i in range(n)]

    def encode_predict_requests_padded(self, model_name: str, inputs: Mapping, shapes: Mapping, *, model_version: Optional[int] = None,
                                       broadcast: Optional[Mapping] = None, order="deterministic", wire_dtype=None,
                                       tensor_content: bool = False, keep_snan: bool = False, grpc_frame: bool = False,
                                       out=None, signature_name=None, version_label=None, output_filter=None) -> List[bytes]:
        """n PredictRequests cut out of one padded tensor per input - the inverse of ``decode_predict_responses_padded``.

        ``inputs[key]`` is a padded tensor ``P`` of shape ``[R, D_1, ..., D_{m-1}]``; ``shapes[key]`` gives each request's shape for it,
        ``int64[n, m]``, or ``int64[n]`` row counts (every trailing dim full).  Request r gets ``P[r0:r0 + S[r,0], :S[r,1], ...,
        :S[r,m-1]]`` with ``r0 = S[:r, 0].sum()``, plus every ``broadcast`` tensor as it is; its bytes are what
        ``encode_predict_request`` returns for that request.  Inputs and shapes may be numpy arrays (pageable or ``pinned_empty``) or
        device arrays (``__cuda_array_interface__`` / DLPack); device shapes never travel to the host - the rows, boxes and framing
        are planned by kernels.  A negative dim, a trailing dim past ``D_j``, a shape of another rank, rows past ``R`` or a request
        count that differs between keys raise ValueError.  ``out="pinned"`` as for ``encode_predict_requests``.

        A string input is a ``BytesColumn`` (padded or broadcast, its data and offsets on the host or the device): each string of a
        box becomes one ``string_val`` value of its raw bytes (NULs and high bytes kept), cut and framed on the device beside the
        numeric inputs; ``wire_dtype`` other than DT_STRING for it raises ValueError.  The offsets a request reads - its first row's
        start, both ends of every string of its box, its last row's end (a broadcast column: every offset) - must never decrease and
        stay within ``0..data_len``.  Host offsets are checked over the whole column before anything runs; device offsets are checked
        by the kernels, only where a box reads them; either way a break raises ValueError.  Numpy str / bytes / object inputs, more
        than 8 padded or 8 broadcast inputs and ranks above 16 are cut on the host and encoded request by request.

        ``signature_name``, ``version_label`` and ``output_filter`` as for ``encode_predict_requests``: the same for every request.
        """
        if out is not None and out != "pinned":
            raise ValueError('out must be None or "pinned"')
        named = dict(signature_name=signature_name, version_label=version_label, output_filter=output_filter)
        spec = _RequestSpec.of([model_version], **named)
        broadcast = dict(broadcast or {})
        if set(inputs) != set(shapes):
            raise ValueError("shapes must have exactly the keys of inputs")
        if set(inputs) & set(broadcast):
            raise ValueError("a key cannot be both padded and broadcast")
        def dims_of(v):
            return v.shape if isinstance(v, BytesColumn) else tuple(D.device_view(v)[1]) if D.is_device_object(v) else np.shape(v)

        pdims = {k: dims_of(v) for k, v in inputs.items()}
        for k, v in list(inputs.items()) + list(broadcast.items()):
            if isinstance(v, BytesColumn):
                _string_wire_dtype(k, wire_dtype.get(k) if isinstance(wire_dtype, Mapping) else wire_dtype)
                _check_host_offsets(k, v)
        n = None
        host_shapes = {}
        for k, s in shapes.items():
            m = len(pdims[k])
            if m < 1:
                raise ValueError(f"input {k!r}: a padded tensor has rank >= 1")
            shp = tuple(D.device_view(s)[1]) if D.is_device_object(s) else np.shape(s)
            if len(shp) not in (1, 2) or (len(shp) == 2 and shp[1] != m):
                raise ValueError(f"shapes of {k!r}: expected int64[n, {m}] or int64[n], got {shp}")
            if n is not None and shp[0] != n:
                raise ValueError(f"shapes of {k!r} give {shp[0]} requests, another key {n}")
            n = shp[0]
            if not D.is_device_object(s):
                a = np.asarray(s)
                if a.dtype.kind not in "iu":
                    raise ValueError(f"shapes of {k!r} must be integers")
                a = a.astype(np.int64).reshape(n, -1)
                if (a < 0).any():
                    raise ValueError(f"shapes of {k!r}: negative dim")
                if a.shape[1] > 1 and (a[:, 1:] > np.asarray(pdims[k][1:], dtype=np.int64)).any():
                    raise ValueError(f"shapes of {k!r}: a trailing dim exceeds the padded tensor's {pdims[k][1:]}")
                if int(a[:, 0].sum()) > pdims[k][0]:
                    raise ValueError(f"shapes of {k!r}: {int(a[:, 0].sum())} rows of {pdims[k][0]}")
                host_shapes[k] = a
        if not n:
            return []
        dtypes = [D.device_view(v)[2] if D.is_device_object(v) else np.asarray(v).dtype for v in list(inputs.values()) + list(broadcast.values())
                  if not isinstance(v, BytesColumn)]
        ranks = list(pdims.values()) + [dims_of(v) for v in broadcast.values()]
        if (any(dt.kind in "OUS" for dt in dtypes) or len(inputs) > N.CONCAT_MAX_KEYS or len(broadcast) > N.CONCAT_MAX_KEYS
                or any(len(r) > N.MAX_RANK for r in ranks)):
            return self._padded_requests_on_host(model_name, model_version, inputs, shapes, broadcast, n, order=order, wire_dtype=wire_dtype,
                                                 tensor_content=tensor_content, keep_snan=keep_snan, grpc_frame=grpc_frame, out=out, **named)
        keep = []

        def dev(v):
            if D.is_device_object(v):
                return v
            a = np.asarray(v)
            if not a.dtype.isnative:
                a = a.astype(a.dtype.newbyteorder("="))
            d = self.device_array(a)
            keep.append(d)
            return d

        preps, pins, strs = [], [], []
        for k, v in list(inputs.items()) + list(broadcast.items()):
            kb = k.encode("utf-8") if isinstance(k, str) else bytes(k)
            wd = wire_dtype.get(k) if isinstance(wire_dtype, Mapping) else wire_dtype
            if isinstance(v, BytesColumn):
                p, b = self._padded_string_input(v, kb, keep)
                strs.append(b)
            else:
                p = _Prepared(dev(v), kb, wd, tensor_content, keep_snan)
                strs.append(N.Bytes())
            if k in broadcast:
                p.struct.flags |= N.F_BROADCAST
                pins.append(N.PadInput(shapes=None, cols=0))
            else:
                s = shapes[k]
                sd = dev(host_shapes[k]) if k in host_shapes else s
                ptr, shp, sdt, hold = D.device_view(sd)
                if sdt != np.int64:
                    raise ValueError(f"device shapes of {k!r} must be int64")
                keep.append(hold)
                pins.append(N.PadInput(shapes=ptr, cols=shp[1] if len(shp) == 2 else 1))
            preps.append(p)
        arr = (N.Tensor * len(preps))(*[p.struct for p in preps])
        pin_arr = (N.PadInput * len(pins))(*pins)
        name = model_name.encode("utf-8") if isinstance(model_name, str) else bytes(model_name)
        order_code = _ORDER[order] if isinstance(order, str) else int(order)
        req = N.Request(model_name=name, model_name_len=len(name), has_version=int(model_version is not None), order=order_code,
                        version=int(model_version) if model_version is not None else 0, n_inputs=len(preps),
                        flags=N.RF_GRPC_FRAME if grpc_frame else 0, inputs=arr)
        cap = C.c_uint64()
        bs = (N.Bytes * len(strs))(*strs) if any(b.offsets for b in strs) else None
        sp = None if spec is None else C.byref(spec.struct)
        N.check(self._lib.b200tfs_padded_request_columns_arena_size_spec(n, C.byref(req), bs, sp, C.byref(cap)))
        if self._pe_arena is None or self._pe_arena.nbytes < cap.value:
            if self._pe_arena is not None:
                self._pe_arena.free()
            self._pe_arena = D.DeviceArray(self, (max(int(cap.value), 1),), np.uint8)
        N.check(self._lib.b200tfs_encode_padded_requests_columns_async_spec(self._ctx, n, C.byref(req), pin_arr, bs, sp, self._pe_arena.ptr,
                                                                             cap.value))
        off, ln = (C.c_uint64 * n)(), (C.c_uint64 * n)()
        rc = self._lib.b200tfs_encode_results(self._ctx, n, off, ln)
        if rc in (N.E_SHAPE, N.E_SIZE):
            raise ValueError(N.last_error())
        N.check(rc)
        end = max(int(off[i]) + int(ln[i]) for i in range(n))
        pw = self._pinned_wire(end)
        if end:
            N.check(self._lib.b200tfs_memcpy_d2h(self._ctx, pw.ptr, self._pe_arena.ptr, end))
        self.sync()
        self.padded_encode_device_calls += 1
        if out == "pinned":
            return [pw.array[off[i]: off[i] + ln[i]] for i in range(n)]
        return [pw.array[off[i]: off[i] + ln[i]].tobytes() for i in range(n)]

    def _padded_string_input(self, col: "BytesColumn", key: bytes, keep: list):
        """(_Prepared-like holder of the DT_STRING Tensor, Bytes entry) of a string column of the padded encode; host arrays are
        copied to the device (the kernels read both there)."""
        data, b = col._bind(keep, upload=self)
        p = _PaddedString(key, col.shape)
        p.struct = N.Tensor(data=data, src_dtype=DT_STRING, wire_dtype=DT_STRING, rank=len(col.shape), flags=N.F_DEVICE_DATA,
                            dims=p.dims, key=key, key_len=len(key), packed_len=0)
        return p, b

    def _to_host(self, v) -> np.ndarray:
        if isinstance(v, BytesColumn):
            if not (v.data_on_device or v.offsets_on_device):
                return v
            data = self._to_host(v.data) if v.data_on_device else v.data
            return BytesColumn(data, self._to_host(v.offsets) if v.offsets_on_device else v.offsets, v.shape)
        if not D.is_device_object(v):
            return np.asarray(v)
        ptr, shape, dtype, _hold = D.device_view(v)
        a = np.empty(shape, dtype=dtype)
        if a.nbytes:
            N.check(self._lib.b200tfs_memcpy_d2h(self._ctx, a.ctypes.data, ptr, a.nbytes))
            self.sync()
        return a

    def _padded_requests_on_host(self, model_name, model_version, inputs, shapes, broadcast, n, **kw) -> List[bytes]:
        """The definition of ``encode_predict_requests_padded``, run on the host: each request's boxes sliced, then encoded."""
        P = {k: self._to_host(v) for k, v in inputs.items()}
        S = {k: self._to_host(s).astype(np.int64).reshape(n, -1) for k, s in shapes.items()}
        B = {k: self._to_host(v) for k, v in broadcast.items()}
        for k, v in B.items():
            if isinstance(v, BytesColumn):
                _check_host_offsets(k, v)   # a broadcast column is read in full; a padded one box by box (_bytes_box)
        for k, s in S.items():
            if (s < 0).any() or (s.shape[1] > 1 and (s[:, 1:] > np.asarray(P[k].shape[1:])).any()) or int(s[:, 0].sum()) > P[k].shape[0]:
                raise ValueError(f"shapes of {k!r} do not fit the padded tensor {P[k].shape}")
        r0 = {k: np.concatenate([[0], np.cumsum(s[:, 0])]) for k, s in S.items()}
        reqs = []
        for r in range(n):
            d = {}
            for k, p in P.items():
                s = S[k][r]
                box = (slice(int(r0[k][r]), int(r0[k][r]) + int(s[0])),) + tuple(slice(0, int(x)) for x in s[1:])
                d[k] = _bytes_box(k, p, int(r0[k][r]), s) if isinstance(p, BytesColumn) else p[box]
            d.update(B)
            reqs.append((model_name, model_version, d))
        return self.encode_predict_requests(reqs, **kw)

    def encode_predict_request(self, model_name: str, input_dict: Mapping, model_version: Optional[int] = None, **kw) -> bytes:
        return self.encode_predict_requests([(model_name, model_version, input_dict)], **kw)[0]

    def encode_example_requests(self, requests: Iterable[Tuple], *, order="deterministic",
                                grpc_frame: bool = False, predict_input=None, tasks=None, signature_name=None, version_label=None,
                                output_filter=None) -> List[bytes]:
        """Each item is ``(model_name, model_version, input_dict)``; returns one ClassificationRequest / RegressionRequest wire
        per item (the two messages share their field numbers, so the bytes serve both RPCs).  With ``predict_input`` (a str or
        bytes key) each wire is instead a PredictRequest for a model that parses serialized tf.Examples: its one input of that
        key is a DT_STRING tensor of shape ``[n]`` whose ``string_val`` holds every example, serialized as the protobuf runtime
        serializes it with ``deterministic=True``.

        An item may also be ``(model_name, model_version, input_dict, context_dict)`` (``None``: no context), in the same call
        as the others: the request then carries an ExampleListWithContext, its examples plus one context Example shared by all
        of them (``examples_with_context_from_input_dict``: the whole of ``context_dict[k]`` is context feature k), the form a
        ranking model takes.  It is the Classify / Regress request's input, or with ``predict_input`` the one string of a
        DT_STRING ``[1]`` tensor (TF-Ranking's serving input).  Context values are taken as input values are, but a
        ``RaggedColumn`` raises ValueError.

        The bytes equal ``_make_example_request(...).SerializeToString(deterministic=True)`` of the request
        ``examples_from_input_dict`` builds - one tf.Example per row, 0-d arrays repeated in every example - with
        ``order="deterministic"``, or list every example's features in insertion order with ``order="given"``.  Values may be
        numpy arrays (pageable or ``pinned_empty``) or device arrays (``__cuda_array_interface__`` / DLPack), and a value may be a
        ``RaggedColumn``: example i then holds only the first ``lengths[i]`` steps of its padded row (device lengths out of range
        raise ValueError).  String features are encoded on the device from a ``BytesColumn`` (offsets that break its rule raise
        ValueError), which ``BytesColumn.from_array`` makes of a numpy str / bytes array.  A request with a numpy str / bytes
        column (or a dtype the device route does not take) is assembled on the host by ``examples_from_input_dict``, in
        deterministic order; device arrays of such dtypes raise ValueError.

        With ``tasks`` - a sequence of ``(signature_name, method_name)``, method_name ``CLASSIFY_METHOD_NAME`` or
        ``REGRESS_METHOD_NAME`` (requests.py) - every wire is instead the MultiInferenceRequest ``make_multi_inference_request``
        builds: one InferenceTask per task, each naming the item's model and version and the task's signature (an empty or None
        one: the server's default), over the Input the item has without tasks.  ``tasks`` with ``predict_input`` raises ValueError.

        ``signature_name`` and ``version_label`` set those model_spec fields of every request (with ``tasks``: the label goes into
        every task's model_spec, and ``signature_name`` raises ValueError, since each task names its own); ``output_filter`` sets
        the PredictRequest's output_filter and needs ``predict_input`` (ValueError otherwise).  A label beside a ``model_version``
        and bytes that are not UTF-8 raise ValueError; None leaves a field unset, and the bytes are those of a call without it.
        """
        items = list(requests)
        fields = {k: v for k, v in dict(signature_name=signature_name, version_label=version_label, output_filter=output_filter).items()
                  if v is not None}
        if output_filter is not None and predict_input is None:
            raise ValueError("output_filter is a PredictRequest field: it needs predict_input (a Classify, Regress or MultiInference "
                             "request has none)")
        if signature_name is not None and tasks is not None:
            raise ValueError("a MultiInference request names a signature per task, not one for the whole request")
        spec = _RequestSpec.of([item[1] for item in items], signature_name, version_label, output_filter)
        order_code = _ORDER[order] if isinstance(order, str) else int(order)
        task_arr = None
        if tasks is not None:
            from .requests import _checked_tasks

            if predict_input is not None:
                raise ValueError("tasks make a MultiInferenceRequest, which carries an Input, not a Predict input")
            tasks = _checked_tasks(tasks)
            sigs = [s.encode("utf-8") for s, _ in tasks]
            task_arr = (N.InferenceTask * len(tasks))(*[N.InferenceTask(signature_name=s, signature_len=len(s),
                                                                        method=N.RESP_CLASSIFY if m == _CLASSIFY_NAME else N.RESP_REGRESS)
                                                        for s, (_, m) in zip(sigs, tasks)])
        pkey = None
        if predict_input is not None:
            pkey = predict_input.encode("utf-8") if isinstance(predict_input, str) else bytes(predict_input)
        out: List[Optional[bytes]] = [None] * len(items)
        keep, structs, dev_idx, ragged, strs, targets, contexts, ctx_strs = [], [], [], [], [], [], [], []
        for i, item in enumerate(items):
            model_name, model_version, input_dict = item[:3]
            context_dict = item[3] if len(item) > 3 else None
            cols = _example_columns(input_dict)
            ccols = _example_columns(context_dict, context=True) if context_dict is not None else None
            if cols is None or (context_dict is not None and ccols is None):
                out[i] = _host_example_request(model_name, model_version, input_dict, grpc_frame, predict_input, context_dict, tasks,
                                               **fields)
                continue
            n, preps = cols
            if ccols is None:
                contexts.append(N.ExampleContext())
            else:
                cpreps = ccols[1]
                cfeats = (N.Feature * max(len(cpreps), 1))(*[p[0] for p in cpreps])
                keep.append((cpreps, cfeats))
                contexts.append(N.ExampleContext(features=cfeats, n_features=len(cpreps), present=1))
                ctx_strs += [p.bytes_entry or N.Bytes() for p in cpreps]
            if pkey is not None:
                kind = N.EXAMPLES_PREDICT_STRING if ccols is None else N.EXAMPLES_PREDICT_ELWC
                targets.append(N.ExampleTarget(kind=kind, key=pkey, key_len=len(pkey)))
            feats = (N.Feature * max(len(preps), 1))(*[p[0] for p in preps])
            name = model_name.encode("utf-8") if isinstance(model_name, str) else bytes(model_name)
            structs.append(N.ExampleRequest(model_name=name, model_name_len=len(name), has_version=int(model_version is not None),
                                            order=order_code, version=int(model_version) if model_version is not None else 0,
                                            n_examples=n, n_features=len(preps), flags=N.RF_GRPC_FRAME if grpc_frame else 0,
                                            features=feats))
            keep.append((preps, feats, name))
            ragged += [p[3] or N.Ragged() for p in preps]
            strs += [p.bytes_entry or N.Bytes() for p in preps]
            dev_idx.append(i)
        if dev_idx:
            m = len(dev_idx)
            reqs = (N.ExampleRequest * m)(*structs)
            cap = C.c_uint64()
            tg = (N.ExampleTarget * m)(*targets) if targets else None
            bs = (N.Bytes * len(strs))(*strs) if any(b.offsets for b in strs) else None
            ct = (N.ExampleContext * m)(*contexts) if any(c.present for c in contexts) else None
            cb = (N.Bytes * len(ctx_strs))(*ctx_strs) if any(b.offsets for b in ctx_strs) else None
            tk = None
            if task_arr is not None:
                tk = (N.ExampleTasks * m)(*[N.ExampleTasks(tasks=C.addressof(task_arr), n_tasks=len(task_arr))] * m)
            rg = (N.Ragged * len(ragged))(*ragged) if any(g.lengths for g in ragged) else None
            specs = _RequestSpec.array(spec, m)
            N.check(self._lib.b200tfs_example_specs_arena_size(m, reqs, None, bs, tg, ct, cb, tk, None, specs, C.byref(cap)))
            wire = np.empty(max(int(cap.value), 1), dtype=np.uint8)
            off, ln = (C.c_uint64 * m)(), (C.c_uint64 * m)()
            N.check(self._lib.b200tfs_encode_example_specs_host(self._ctx, m, reqs, rg, bs, tg, ct, cb, tk, None, specs, wire.ctypes.data,
                                                                cap.value, off, ln))
            for j, i in enumerate(dev_idx):
                out[i] = wire[off[j]: off[j] + ln[j]].tobytes()
        return out  # type: ignore[return-value]

    def encode_sequence_example_requests(self, requests: Iterable[Tuple], *, input_key, order="deterministic",
                                         grpc_frame: bool = False, signature_name=None, version_label=None,
                                         output_filter=None) -> List[bytes]:
        """Each item is ``(model_name, model_version, context_dict, feature_list_dict)``; returns one PredictRequest wire per item
        for a model that parses serialized tf.SequenceExamples: its one input ``input_key`` is the DT_STRING ``[n]`` tensor of the
        sequences ``requests.sequence_examples_from_input_dict`` builds, each serialized with ``deterministic=True`` - the bytes of
        ``make_predict_sequence_examples_request(...).SerializeToString(deterministic=True)``.

        Context values are taken as ``encode_example_requests`` takes input values (row i is sequence i's; 0-d values repeated;
        ``RaggedColumn`` and ``BytesColumn``).  A feature-list value has shape ``[n, T, *inner]``: a numpy, pinned or device
        array, a ``BytesColumn``, or a ``RaggedColumn`` of either whose sequence i has ``lengths[i]`` steps (device lengths out of
        range raise ValueError); step t of sequence i is one Feature of ``value[i, t]``.  ``order="given"`` lists the context and
        the feature lists in insertion order.  An item with a numpy str / bytes value, or a dtype the device route does not take,
        is assembled on the host by ``make_predict_sequence_examples_request`` (deterministic order); device arrays of such dtypes
        raise ValueError.  ``signature_name``, ``version_label`` and ``output_filter`` as for ``encode_predict_requests``."""
        from .requests import make_predict_sequence_examples_request

        items = list(requests)
        fields = {k: v for k, v in dict(signature_name=signature_name, version_label=version_label, output_filter=output_filter).items()
                  if v is not None}
        spec = _RequestSpec.of([item[1] for item in items], signature_name, version_label, output_filter)
        order_code = _ORDER[order] if isinstance(order, str) else int(order)
        pkey = input_key.encode("utf-8") if isinstance(input_key, str) else bytes(input_key)
        out: List[Optional[bytes]] = [None] * len(items)
        keep, structs, dev_idx, ragged, strs, targets, seqs = [], [], [], [], [], [], []
        for i, (model_name, model_version, context_dict, feature_list_dict) in enumerate(items):
            n = _sequence_count(context_dict, feature_list_dict)
            ccols, lcols = _example_columns(context_dict), _example_columns(feature_list_dict)
            if ccols is None or lcols is None:
                req = make_predict_sequence_examples_request(model_name, model_version, context_dict, feature_list_dict, pkey.decode("utf-8"),
                                                             **fields)
                wire = req.SerializeToString(deterministic=True)
                out[i] = (b"\x00" + len(wire).to_bytes(4, "big") + wire) if grpc_frame else wire
                continue
            cpreps, lpreps = ccols[1], lcols[1]
            # a feature list's steps: T and the elements of one step, from its padded shape
            lrag = []
            for p, v in zip(lpreps, feature_list_dict.values()):
                shape = _shape_of(v)
                g = p[3] or N.Ragged()
                g.max_len, g.unit = shape[1], int(np.prod(shape[2:], dtype=np.int64))
                lrag.append(g)
            preps = cpreps + lpreps
            feats = (N.Feature * max(len(preps), 1))(*[p[0] for p in preps])
            name = model_name.encode("utf-8") if isinstance(model_name, str) else bytes(model_name)
            structs.append(N.ExampleRequest(model_name=name, model_name_len=len(name), has_version=int(model_version is not None),
                                            order=order_code, version=int(model_version) if model_version is not None else 0,
                                            n_examples=n, n_features=len(preps), flags=N.RF_GRPC_FRAME if grpc_frame else 0,
                                            features=feats))
            keep.append((preps, feats, name))
            ragged += [p[3] or N.Ragged() for p in cpreps] + lrag
            strs += [p.bytes_entry or N.Bytes() for p in preps]
            targets.append(N.ExampleTarget(kind=N.EXAMPLES_PREDICT_SEQUENCE, key=pkey, key_len=len(pkey)))
            seqs.append(N.ExampleSequence(present=1, n_context=len(cpreps)))
            dev_idx.append(i)
        if dev_idx:
            m = len(dev_idx)
            reqs = (N.ExampleRequest * m)(*structs)
            tg, sq = (N.ExampleTarget * m)(*targets), (N.ExampleSequence * m)(*seqs)
            rg = (N.Ragged * max(len(ragged), 1))(*ragged)
            bs = (N.Bytes * len(strs))(*strs) if any(b.offsets for b in strs) else None
            cap = C.c_uint64()
            specs = _RequestSpec.array(spec, m)
            N.check(self._lib.b200tfs_example_specs_arena_size(m, reqs, rg, bs, tg, None, None, None, sq, specs, C.byref(cap)))
            wire = np.empty(max(int(cap.value), 1), dtype=np.uint8)
            off, ln = (C.c_uint64 * m)(), (C.c_uint64 * m)()
            N.check(self._lib.b200tfs_encode_example_specs_host(self._ctx, m, reqs, rg, bs, tg, None, None, None, sq, specs, wire.ctypes.data,
                                                                cap.value, off, ln))
            for j, i in enumerate(dev_idx):
                out[i] = wire[off[j]: off[j] + ln[j]].tobytes()
        return out  # type: ignore[return-value]

    def encode_elwc_requests(self, requests: Iterable[Tuple], *, input_key, order="deterministic", grpc_frame: bool = False,
                             signature_name=None, version_label=None, output_filter=None) -> List[bytes]:
        """Each item is ``(model_name, model_version, context_dict, input_dict, list_sizes)``; returns one PredictRequest wire per
        item for a TF-Ranking model whose ELWC signature takes a DT_STRING ``[Q]`` vector of serialized ExampleListWithContexts,
        one per query - the bytes of ``make_predict_elwcs_request(...).SerializeToString(deterministic=True)``.  ``list_sizes``
        (host integers, Q of them) cuts the rows of ``input_dict`` into the queries' candidate lists; row q of ``context_dict`` is
        query q's context.

        Values are taken as ``encode_sequence_example_requests`` takes context values (numpy, pinned or device arrays, 0-d values
        repeated, ``RaggedColumn`` and ``BytesColumn``), on both sides.  ``order="given"`` lists the features in insertion order.
        An item with a numpy str / bytes value, or a dtype the device route does not take, is assembled on the host by
        ``make_predict_elwcs_request`` (deterministic order); device arrays of such dtypes raise ValueError, and so do device
        lengths or offsets out of range.  ``signature_name``, ``version_label`` and ``output_filter`` as for
        ``encode_predict_requests``.  With one query the bytes equal ``encode_example_requests(..., predict_input=input_key)``'s
        for that query's context.

        ``list_sizes`` may also be a device int64 vector (``__cuda_array_interface__`` / DLPack), which the host never reads: the
        rows of ``input_dict`` are then a capacity N, the sizes may add up to any total <= N, and the rows from the total on are not
        sent - what a GPU retrieval or filtering stage leaves, a flat candidate buffer and per-query counts.  The rows past the
        total are still counted, so ragged lengths and string offsets there must keep the rules (length 0, or offsets equal to
        the last used one, do).  A negative size or a total past N raises ValueError from the encode; so do a device int32 vector
        and an item whose input values are all 0-d (it has no capacity).  An item the host assembles copies the sizes to the host
        and cuts the rows to their total."""
        from .requests import _list_sizes, make_predict_elwcs_request

        items = list(requests)
        fields = {k: v for k, v in dict(signature_name=signature_name, version_label=version_label, output_filter=output_filter).items()
                  if v is not None}
        spec = _RequestSpec.of([item[1] for item in items], signature_name, version_label, output_filter)
        order_code = _ORDER[order] if isinstance(order, str) else int(order)
        pkey = input_key.encode("utf-8") if isinstance(input_key, str) else bytes(input_key)
        out: List[Optional[bytes]] = [None] * len(items)
        keep, structs, dev_idx, ragged, strs, lists, lragged, lstrs, dlists = [], [], [], [], [], [], [], [], []
        for i, (model_name, model_version, context_dict, input_dict, list_sizes) in enumerate(items):
            dsizes = None        # device list sizes: (pointer, keep-alive)
            if D.is_device_object(list_sizes):
                ptr, sshape, sdtype, shold = D.device_view(list_sizes)
                if sdtype != np.int64 or len(sshape) != 1:
                    raise ValueError(f"device list sizes must be an int64 vector, got {sdtype} of shape {tuple(sshape)}")
                rows = {_shape_of(v)[0] for v in input_dict.values() if len(_shape_of(v))}
                if not rows:
                    raise ValueError("device list sizes need an input value with a row axis: its rows are the candidate capacity")
                if len(rows) > 1:
                    raise ValueError(f"inputs disagree on the number of rows: {sorted(rows)}")
                n, q = rows.pop(), int(sshape[0])
                dsizes, sizes = (ptr, shold), None
            else:
                sizes = _list_sizes(list_sizes)
                n, q = int(sizes.sum()), sizes.size
            for what, d, m in (("input", input_dict, n), ("context", context_dict, q)):
                for k, v in d.items():
                    shape = _shape_of(v)
                    if len(shape) and shape[0] != m:
                        raise ValueError(f"{what} {k!r} has {shape[0]} rows, not {m}")
            on_device = dsizes is not None
            if on_device and not q:     # no size to read (an empty vector may have no address): no row is sent
                dsizes, sizes, n = None, np.zeros(0, np.int64), 0
            cols, ccols = _example_columns(input_dict), _example_columns(context_dict)
            if cols is None or ccols is None or (n and not input_dict):
                if on_device:
                    if dsizes is not None:
                        sizes = np.empty(q, dtype=np.int64)
                        N.check(self._lib.b200tfs_memcpy_d2h(self._ctx, sizes.ctypes.data, dsizes[0], sizes.nbytes))
                        self.sync()
                    if (sizes < 0).any() or int(sizes.sum()) > n:
                        raise ValueError(f"list sizes must be >= 0 and add up to at most the {n} rows")
                    input_dict = {k: _head_rows(v, int(sizes.sum())) for k, v in input_dict.items()}
                req = make_predict_elwcs_request(model_name, model_version, context_dict, input_dict, sizes, pkey.decode("utf-8"), **fields)
                wire = req.SerializeToString(deterministic=True)
                out[i] = (b"\x00" + len(wire).to_bytes(4, "big") + wire) if grpc_frame else wire
                continue
            preps, cpreps = cols[1], ccols[1]
            feats = (N.Feature * max(len(preps), 1))(*[p[0] for p in preps])
            cfeats = (N.Feature * max(len(cpreps), 1))(*[p[0] for p in cpreps])
            name = model_name.encode("utf-8") if isinstance(model_name, str) else bytes(model_name)
            structs.append(N.ExampleRequest(model_name=name, model_name_len=len(name), has_version=int(model_version is not None),
                                            order=order_code, version=int(model_version) if model_version is not None else 0,
                                            n_examples=n, n_features=len(preps), flags=N.RF_GRPC_FRAME if grpc_frame else 0,
                                            features=feats))
            lists.append(N.ExampleLists(list_sizes=sizes.ctypes.data if q and dsizes is None else None, n_lists=q, context=cfeats,
                                        n_context=len(cpreps), present=1))
            dlists.append(N.ExampleDeviceLists(sizes=dsizes[0] or None) if dsizes is not None else N.ExampleDeviceLists())
            keep.append((preps, feats, cpreps, cfeats, name, sizes, dsizes))
            ragged += [p[3] or N.Ragged() for p in preps]
            strs += [p.bytes_entry or N.Bytes() for p in preps]
            lragged += [p[3] or N.Ragged() for p in cpreps]
            lstrs += [p.bytes_entry or N.Bytes() for p in cpreps]
            dev_idx.append(i)
        if dev_idx:
            m = len(dev_idx)
            reqs = (N.ExampleRequest * m)(*structs)
            tg = (N.ExampleTarget * m)(*[N.ExampleTarget(kind=N.EXAMPLES_PREDICT_ELWCS, key=pkey, key_len=len(pkey))] * m)
            ls = (N.ExampleLists * m)(*lists)
            rg = (N.Ragged * len(ragged))(*ragged) if any(g.lengths for g in ragged) else None
            bs = (N.Bytes * len(strs))(*strs) if any(b.offsets for b in strs) else None
            lrg = (N.Ragged * len(lragged))(*lragged) if any(g.lengths for g in lragged) else None
            lbs = (N.Bytes * len(lstrs))(*lstrs) if any(b.offsets for b in lstrs) else None
            dls = (N.ExampleDeviceLists * m)(*dlists) if any(d.sizes for d in dlists) else None
            cap = C.c_uint64()
            specs = _RequestSpec.array(spec, m)
            N.check(self._lib.b200tfs_example_device_lists_arena_size(m, reqs, None, bs, tg, None, None, None, None, specs, ls, lrg, lbs,
                                                                      dls, C.byref(cap)))
            wire = np.empty(max(int(cap.value), 1), dtype=np.uint8)
            off, ln = (C.c_uint64 * m)(), (C.c_uint64 * m)()
            N.check(self._lib.b200tfs_encode_example_device_lists_host(self._ctx, m, reqs, rg, bs, tg, None, None, None, None, specs, ls,
                                                                       lrg, lbs, dls, wire.ctypes.data, cap.value, off, ln))
            for j, i in enumerate(dev_idx):
                out[i] = wire[off[j]: off[j] + ln[j]].tobytes()
        return out  # type: ignore[return-value]

    # ---- decode --------------------------------------------------------------------------------
    def _pack_wires(self, wires: Sequence[bytes]):
        n = len(wires)
        off = (C.c_uint64 * max(n, 1))()
        ln = (C.c_uint64 * max(n, 1))()
        if n == 1 and len(wires[0]) and (isinstance(wires[0], (bytes, bytearray, memoryview)) or
                                         (isinstance(wires[0], np.ndarray) and wires[0].dtype == np.uint8 and wires[0].flags.c_contiguous)):
            # a single message: hand its own buffer to the library (read-only view, no copy)
            view = wires[0] if isinstance(wires[0], np.ndarray) else np.frombuffer(wires[0], dtype=np.uint8)
            ln[0] = view.size
            return view, off, ln
        cur = 0
        for i, w in enumerate(wires):
            off[i] = cur
            ln[i] = len(w)
            cur += (len(w) + 255) & ~255  # records start 256-byte aligned, like a received buffer would
        buf = np.empty(max(cur, 1), dtype=np.uint8)
        for i, w in enumerate(wires):
            if len(w):
                buf[off[i]: off[i] + len(w)] = w if isinstance(w, np.ndarray) else np.frombuffer(w, dtype=np.uint8)
        return buf, off, ln

    @staticmethod
    def _text(buf: np.ndarray, off: int, length: int) -> str:
        return buf[off: off + length].tobytes().decode("utf-8")

    @staticmethod
    def _spec(buf: np.ndarray, base: int, s: N.ModelSpec) -> "DecodedSpec":
        """The model_spec of the record at `base` (the table's offsets are record-relative)."""
        t = Codec._text
        return DecodedSpec(t(buf, base + s.name_off, s.name_len), int(s.version), bool(s.has_version),
                           t(buf, base + s.label_off, s.label_len), t(buf, base + s.signature_off, s.signature_len))

    @staticmethod
    def _table(buf: np.ndarray, off, outs, n_outs, width: int, i: int) -> Dict[str, N.Output]:
        """{key: Output} of record i, from a table of `width` entries per record (its offsets are relative to the record)."""
        base = int(off[i])
        return {Codec._text(buf, base + o.key_off, o.key_len): o for o in (outs[i * width + j] for j in range(n_outs[i]))}

    def _unpack_to_host(self, jobs):
        """b200tfs_unpack_outputs_host over (into, key, Output, numpy type, dst dtype code, shape, record offset) jobs, the
        record offsets into the staged wire: one new array per job, stored at ``into[key]``.  The first job that failed
        raises - ValueError when the values do not fill the shape."""
        m = len(jobs)
        if not m:
            return
        arrays = [np.empty(j[5], dtype=j[3]) for j in jobs]
        outs = (N.Output * m)(*[j[2] for j in jobs])
        dst = (C.c_void_p * m)(*[a.ctypes.data if a.size else None for a in arrays])
        codes = (C.c_int32 * m)(*[j[4] for j in jobs])
        status = (C.c_int32 * m)()
        rec = (C.c_uint64 * m)(*[j[6] for j in jobs])
        N.check(self._lib.b200tfs_unpack_outputs_host(self._ctx, m, outs, rec, dst, codes, status))
        for k, j in enumerate(jobs):
            if status[k] == N.E_SHAPE:
                raise ValueError(f"cannot reshape array into shape {j[5]}")
            N.check(status[k])
        for (into, key, *_), a in zip(jobs, arrays):
            into[key] = a

    def parse_predict_responses(self, wires: Sequence[bytes], max_outputs: int = 16) -> List[ParsedResponse]:
        """Run the parse kernel over each PredictResponse; raises DecodeError like ``FromString``.  ``max_outputs`` sizes
        the first attempt only: a response with more outputs is parsed again with a table twice as wide, and so on
        (``PredictResponse.FromString`` has no limit on the map size)."""
        n = len(wires)
        if n == 0:
            return []
        buf, off, ln = self._pack_wires(wires)
        while True:
            outs = (N.Output * (n * max_outputs))()
            n_outs = (C.c_int32 * n)()
            specs = (N.ModelSpec * n)()
            status = (C.c_int32 * n)()
            N.check(self._lib.b200tfs_parse_responses_host(self._ctx, buf.ctypes.data, n, off, ln, max_outputs, outs, n_outs, specs, status))
            if max_outputs < (1 << 20) and any(status[i] == N.E_SIZE for i in range(n)):
                max_outputs *= 2
                continue
            break
        parsed = []
        for i in range(n):
            if status[i] == N.E_SIZE:
                raise ValueError(f"response {i} has more than max_outputs={max_outputs} outputs")
            if status[i] != N.OK:
                from google.protobuf.message import DecodeError

                raise DecodeError(f"Error parsing message (response {i}, status {status[i]})")
            table = self._table(buf, off, outs, n_outs, max_outputs, i)
            parsed.append(ParsedResponse(buf, int(off[i]), int(ln[i]), int(status[i]), table, self._spec(buf, int(off[i]), specs[i])))
        return parsed

    def _resolve_output(self, o: N.Output, strict: bool, out_dtype):
        """(numpy dtype, native dst dtype code, shape) for one tabulated output, or raise what the
        reference raises for it (tensors.py:42-46, types.py:39-40)."""
        enum = int(o.dtype)
        if strict and enum == DT_BFLOAT16:
            raise KeyError(enum)  # not in the reference's ENUM_TO_TF_MAPPING
        if o.status == N.E_KEY:
            raise KeyError(enum)
        np_type = numpy_for_enum(enum)
        shape = self._shape(o)
        if (o.flags & N.OF_RANK0) and strict:
            # reshape() with no dims raises whatever the values are, so this comes before any element-count error
            raise TypeError("reshape() takes exactly 1 argument (0 given)")
        if strict and enum in (DT_COMPLEX64, DT_COMPLEX128) and o.n_elems:
            raise ValueError("cannot reshape array: the reference reads complex values as separate floats")
        content_only = o.n_runs == 0 and o.content_len and o.n_strings == 0
        if content_only and not strict and o.content_len == int(np.prod(shape, dtype=np.int64)) * np.dtype(np_type).itemsize:
            pass  # tolerant: raw little-endian tensor_content, as TF writes it
        elif o.status == N.E_SHAPE and not strict and out_dtype is None and self._may_pad(o, np_type):
            # tolerant: TensorFlow's MakeNdarray padding - no values: zeros; fewer than the shape holds: the last one repeats
            o.flags |= N.OF_PAD_EDGE
        elif o.status == N.OK and not strict and out_dtype is None and (o.flags & N.OF_VARINT) and o.n_elems > 0:
            o.flags |= N.OF_PAD_EDGE   # packed varints: whether there are fewer values than elements is only known to the decode kernels
        elif o.status == N.E_SHAPE:
            raise ValueError(f"cannot reshape array into shape {shape}")
        elif o.status == N.E_NONCANONICAL:
            raise NotImplementedError("wire layout not tabulated by the device parser")
        elif o.status != N.OK:
            N.check(o.status)
        dst_code = enum
        if out_dtype is not None:
            dst_code = _as_enum(out_dtype)
            np_type = numpy_for_enum(dst_code)
        elif strict and enum == DT_HALF:
            dst_code = N.DT_HALF_REFQUIRK
        return np_type, dst_code, shape

    def _shape(self, o: N.Output) -> Tuple[int, ...]:
        """Every dim of an output: the table holds MAX_RANK inline, deeper shapes come from the context's spill area."""
        if o.rank <= N.MAX_RANK:
            return tuple(int(o.dims[k]) for k in range(o.rank))
        dims = (C.c_int64 * o.rank)()
        N.check(self._lib.b200tfs_output_dims(self._ctx, C.byref(o), dims, o.rank))
        return tuple(int(d) for d in dims)

    def _runs(self, o: N.Output) -> List[N.Run]:
        """Every value run of an output (inline + spilled), in wire order."""
        if o.n_runs <= o.n_inline:
            return [o.runs[k] for k in range(o.n_runs)]
        runs = (N.Run * o.n_runs)()
        N.check(self._lib.b200tfs_output_runs(self._ctx, C.byref(o), runs, o.n_runs))
        return list(runs)

    def _may_pad(self, o: N.Output, np_type) -> bool:
        """An E_SHAPE output the padding rule applies to: the shape is fully known and holds MORE elements than there are
        values (packed varints: more elements than value bytes would be needed; the kernel then counts exactly)."""
        if o.n_elems <= 0 or o.content_len or any(d < 0 for d in self._shape(o)):
            return False
        value_bytes = sum(int(r.len) * int(r.count) for r in self._runs(o))
        if o.flags & N.OF_VARINT:
            return True     # fewer value bytes than elements was what raised E_SHAPE here; a surplus is caught by the decode kernels
        size = np.dtype(np_type).itemsize
        return value_bytes % size == 0 and value_bytes // size < o.n_elems

    def decode_predict_responses(self, wires: Sequence[bytes], *, strict: bool = False, out_dtypes: Optional[Mapping] = None,
                                 max_outputs: int = 16) -> List[Tuple[Dict[str, np.ndarray], DecodedSpec]]:
        """``PredictResponse.FromString`` + ``tensor_proto_to_ndarray`` on every output, on the GPU.

        ``strict=True`` reproduces the reference's behaviour case for case (including the inputs it
        rejects); the default additionally accepts what TF itself emits: ``tensor_content``, rank-0
        tensors, complex pairs, bfloat16, and reads ``half_val`` as bit patterns.
        """
        fused = None
        if out_dtypes is None and len(wires):
            fused = self._decode_fused(wires, strict)
        elif out_dtypes and len(wires) and not strict and _narrowing_cast(out_dtypes) is not None:
            # every requested cast is the same narrowing of float32 (BASELINE config C4): one launch does it (b200tfs_set_decode_cast)
            fused = self._decode_fused(wires, strict, dict(out_dtypes))
        return fused if fused is not None else self._decode_two_phase(wires, strict, out_dtypes, max_outputs)

    def _decode_two_phase(self, wires, strict, out_dtypes, max_outputs, keys=None, raw_strings=False):
        """The parse kernel, then the unpack of every output - of the outputs named in `keys` only, when given (the others are
        neither converted nor checked).  `raw_strings`: string outputs as _RawStrings instead of numpy str arrays."""
        parsed = self.parse_predict_responses(wires, max_outputs=max_outputs)
        jobs = []
        results: List[Tuple[Dict[str, np.ndarray], DecodedSpec]] = []
        for pr in parsed:
            arrays: Dict[str, np.ndarray] = {}
            results.append((arrays, pr.model_spec))
            for key, o in pr.outputs.items():
                if keys is not None and key not in keys:
                    continue
                if raw_strings and int(o.dtype) == DT_STRING and o.status == N.E_SHAPE:
                    raise ValueError(f"output {key!r}: {int(o.n_strings)} strings do not fill its shape")
                if int(o.dtype) == DT_STRING and o.status == N.OK:
                    if raw_strings:
                        proto = self._string_proto(pr.wire, pr.offset, o, pr.length, key)
                        strs = list(proto.string_val)
                        shape = np.empty(len(strs), np.uint8).reshape(tuple(int(d.size) for d in proto.tensor_shape.dim)).shape
                        arrays[key] = _RawStrings(strs, shape)
                    else:
                        arrays[key] = self._decode_strings(pr.wire, pr.offset, o, pr.length, key)
                    continue
                np_type, dst_code, shape = self._resolve_output(o, strict, out_dtypes.get(key) if out_dtypes else None)
                jobs.append((arrays, key, o, np_type, dst_code, shape, pr.offset))
        self._unpack_to_host(jobs)
        return results

    @contextlib.contextmanager
    def _decode_modes(self, cast_code: int = 0, varints: bool = False):
        """The context's narrowing cast and varint decode switched on for the native calls inside, and off after them."""
        if cast_code:
            N.check(self._lib.b200tfs_set_decode_cast(self._ctx, cast_code))
        if varints:
            N.check(self._lib.b200tfs_set_decode_varints(self._ctx, 1))
        try:
            yield
        finally:
            if cast_code:
                N.check(self._lib.b200tfs_set_decode_cast(self._ctx, 0))
            if varints:
                N.check(self._lib.b200tfs_set_decode_varints(self._ctx, 0))

    def _fused_launch(self, wires: Sequence[bytes], cast_code: int = 0, dst: Optional[np.ndarray] = None,
                      stride: int = 0) -> Optional["_Launch"]:
        """H2D of the wire, decode_fused_kernel, D2H of the decoded fixed-width outputs, one synchronise, into slots sized by
        _slot_stride - or into the caller's page-locked `dst` at `stride`, varint decode off.  None if any record was not
        tabulated (malformed, or more than FUSED_MAX_OUTPUTS outputs)."""
        n = len(wires)
        buf, off, ln = self._pack_wires(wires)
        varints = False
        if dst is None:
            stride, varints = self._slot_stride(buf, off, ln)
            dst = np.empty(n * stride, dtype=np.uint8)
        with self._decode_modes(cast_code, varints):
            N.check(self._lib.b200tfs_decode_responses_host_async(self._ctx, buf.ctypes.data, n, off, ln, dst.ctypes.data, stride))
        outs = (N.Output * (n * N.FUSED_MAX_OUTPUTS))()
        n_outs = (C.c_int32 * n)()
        specs = (N.ModelSpec * n)()
        status = (C.c_int32 * n)()
        N.check(self._lib.b200tfs_decode_results(self._ctx, n, outs, n_outs, specs, status))   # synchronises
        if any(status[i] != N.OK for i in range(n)):
            return None
        tables = [self._table(buf, off, outs, n_outs, N.FUSED_MAX_OUTPUTS, i) for i in range(n)]
        return _Launch(n, buf, off, dst, stride, tables, specs)

    def open_predict_response(self, wire: bytes) -> Optional["OpenResponse"]:
        """Decode one PredictResponse now, hand its outputs out later (``PredictResponseView.outputs``): the launch moves
        every fixed-width output; ``OpenResponse.array(key, strict)`` applies the reference's per-output rules on demand."""
        if not len(wire):
            return None
        launch = self._fused_launch([wire])
        if launch is None:
            return None
        table = launch.tables[0]
        if any(o.n_elems and int(o.dtype) in _VARINT_DTYPES for o in table.values()):
            self._seen_varints = True
        return OpenResponse(self, launch.buf, int(launch.off[0]), launch.dst, table)

    def _slot_stride(self, buf, off, ln) -> Tuple[int, bool]:
        """(dst_stride, decode varints) for the records of ONE call.  Every fixed-width output fits the parent layout's stride
        (longest record + one 256-byte alignment per output).  Once this codec has seen varint outputs, the host walks the
        call's records (b200tfs_decode_slot_bytes) and, when they carry varint outputs, the stride is what their layout with
        varint ranges needs - so a float-only call keeps the plain stride, and a denser response never pushes an output out."""
        n = len(ln)
        stride = (max(int(ln[i]) for i in range(n)) + 256 * (N.FUSED_MAX_OUTPUTS + 1) + 255) & ~255
        if not self._seen_varints:
            return stride, False
        need, nv = C.c_uint64(), C.c_int32()
        N.check(self._lib.b200tfs_decode_slot_bytes(buf.ctypes.data, n, off, ln, 1, C.byref(need), C.byref(nv)))
        if not nv.value:
            return stride, False
        return max(stride, (need.value + 255) & ~255), True

    def _decode_fused(self, wires: Sequence[bytes], strict: bool, cast_keys: Optional[Dict] = None):
        """One launch, one synchronise: tag walk (or framing-template check), destination layout and the move of every
        fixed-width output in ``decode_fused_kernel``; the outputs come back as views of one host buffer.  Once this codec has
        seen varint-packed outputs, the same launch decodes those too (b200tfs_set_decode_varints) and they come back as views
        as well; the ones it cannot finish (TF's padding, strict DT_HALF, rows of unpacked elements, errors) and
        tensor_content-only outputs are unpacked by a second one.  Returns None when
        a record needs the two-phase path (more than eight outputs, a malformed record: that path raises what the
        reference raises).  `cast_keys`: out_dtypes asking for one narrowing of float32 (b200tfs_set_decode_cast)."""
        cast_keys = cast_keys or {}
        cast_code = _narrowing_cast(cast_keys) if cast_keys else 0
        launch = self._fused_launch(wires, cast_code)
        if launch is None:
            return None
        results: List[Tuple[Dict[str, np.ndarray], DecodedSpec]] = []
        jobs = []
        for i in range(launch.n):
            base = int(launch.off[i])
            arrays: Dict[str, np.ndarray] = {}
            results.append((arrays, self._spec(launch.buf, base, launch.specs[i])))
            for key, o in launch.tables[i].items():
                if int(o.dtype) == DT_STRING and o.status == N.OK:
                    arrays[key] = self._decode_strings(launch.buf, base, o, len(wires[i]), key)
                    continue
                if cast_code and not _narrowing_fits(o.dtype, key, cast_keys):
                    return None
                if int(o.dtype) in _VARINT_DTYPES and o.n_elems:
                    self._seen_varints = True
                stored = _stored(o)
                np_type, dst_code, shape = self._resolve_output(o, strict, cast_keys.get(key))
                if stored and _stored_as(o, dst_code, cast_code):
                    at = i * launch.stride + int(o.dst_off)
                    arrays[key] = launch.dst[at: at + int(o.dst_bytes)].view(np_type).reshape(shape)
                else:
                    jobs.append((arrays, key, o, np_type, dst_code, shape, base))
        self._unpack_to_host(jobs)
        return results

    # ---- batch decode into one tensor per key ------------------------------------------------------
    def decode_predict_responses_concat(self, wires: Sequence[bytes], keys: Optional[Sequence[str]] = None, *, strict: bool = False,
                                        out_dtypes: Optional[Mapping] = None, device: bool = False, out: Optional[Mapping] = None,
                                        string_columns: bool = False) -> Tuple[Dict[str, object], List[DecodedSpec]]:
        """Decode a batch of PredictResponses into ONE tensor per output: for every key, the outputs of all responses
        concatenated along axis 0 - ``np.concatenate([decode_predict_responses([w], ...)[0][0][key] for w in wires], axis=0)``,
        bit for bit and with the same exceptions, except that outputs of different dtypes raise ValueError instead of being
        promoted, and that outputs which are not requested are not decoded (an error confined to them does not raise).

        ``keys=None``: every key of the first response.  ``device=True`` returns ``DeviceArray``s (``__cuda_array_interface__``:
        ``torch.as_tensor(a, device="cuda")`` takes them without a copy); otherwise numpy arrays, one device-to-host copy per
        key.  ``out={key: array}`` writes in place: a C-contiguous device array (CUDA array interface / DLPack) or a numpy /
        ``pinned_empty`` array of exactly the result's dtype and shape.  Returns ``({key: tensor}, [DecodedSpec per response])``.

        ``string_columns=True``: every DT_STRING output comes back as a ``BytesColumn`` - the raw bytes of every response's
        ``string_val`` (no UTF-8 check, NULs and high bytes kept), concatenated in response order, with ``offsets`` int64[m + 1]
        from 0 and the concatenated shape - decoded on the device in the same call as the numeric outputs (``DeviceArray`` data and
        offsets with ``device=True``, numpy arrays otherwise).  Such a column feeds ``encode_example_requests`` directly.  ``out``
        naming a string output raises ValueError.  Without it, string outputs are numpy str arrays decoded on the host (and
        ``device=True`` raises TypeError for them).
        """
        buf, off, ln, keys, out_dtypes, out = self._requested(wires, keys, out, out_dtypes, "need at least one response to concatenate")
        fast = self._concat_device(wires, buf, off, ln, keys, strict, out_dtypes, device, out, string_columns)
        if fast is not None:
            return fast
        return self._concat_per_record(wires, keys, strict, out_dtypes, device, out, string_columns)

    def _requested(self, wires, keys, out, out_dtypes, empty: str):
        """The front of a per-key batch decode: the batch staged (_pack_wires), the requested keys (None: every key of the first
        response), out_dtypes restricted to them and `out` as a dict.  ValueError(`empty`) for an empty batch, KeyError for a
        key of `out` that is not requested."""
        if len(wires) == 0:
            raise ValueError(empty)
        out = dict(out or {})
        buf, off, ln = self._pack_wires(wires)
        if keys is None:
            keys = self._response_keys(buf, int(off[0]), int(ln[0]))
            if keys is None:      # the first response does not parse: the parse raises what the reference raises
                self.parse_predict_responses(wires[:1])
                from google.protobuf.message import DecodeError

                raise DecodeError("Error parsing message (response 0)")
        keys = list(dict.fromkeys(keys))
        for k in out:
            if k not in keys:
                raise KeyError(k)
        if out_dtypes:        # only the requested outputs are decoded: entries for other keys play no part
            out_dtypes = {k: v for k, v in out_dtypes.items() if k in keys} or None
        return buf, off, ln, keys, out_dtypes, out

    def _response_keys(self, buf, base: int, length: int) -> Optional[List[str]]:
        cap = 64
        while True:
            ko, kl, cnt = (C.c_uint64 * cap)(), (C.c_uint32 * cap)(), C.c_int32()
            rc = self._lib.b200tfs_response_keys(buf.ctypes.data + base, length, cap, ko, kl, C.byref(cnt))
            if rc != N.OK:
                return None
            if cnt.value <= cap:
                return [self._text(buf, base + int(ko[i]), int(kl[i])) for i in range(cnt.value)]
            cap = cnt.value

    def _per_record(self, wires, keys, strict, out_dtypes, device, out, bad_rank, combine, string_column=None):
        """The definition itself, response by response, for the requested outputs: what a device route hands over when a batch
        holds a case it does not take (a malformed record, more than FUSED_MAX_OUTPUTS outputs or MAX_RANK dims, TF padding,
        tensor_content only, strings, mismatches).  Like the device routes it converts and checks the requested outputs only.
        Per key, the route's rank rule (`bad_rank(key, parts)`: the ValueError's message, or None), one dtype, and the route's
        tensor of the parts (`combine(key, parts)`).  `string_column(key, parts)`: the route's BytesColumn of string outputs, whose
        parts are then _RawStrings of their raw bytes (None: numpy str arrays)."""
        wanted = set(keys)
        per = [self._decode_two_phase([w], strict, out_dtypes, 16, wanted, string_column is not None)[0] for w in wires]
        result = {}
        for k in keys:
            parts = [p[0][k] for p in per]
            if any(isinstance(a, _RawStrings) for a in parts):
                result[k] = string_column(k, parts)
                continue
            msg = bad_rank(k, parts)
            if msg:
                raise ValueError(msg)
            if len({a.dtype for a in parts}) > 1:
                raise ValueError(f"output {k!r}: responses disagree on the dtype ({', '.join(sorted({str(a.dtype) for a in parts}))})")
            arr = combine(k, parts)
            if device and arr.dtype.kind in "US":
                raise TypeError(f"output {k!r}: string tensors are decoded on the host")
            result[k] = self._concat_deliver(k, arr, device, out)
        return result, [p[1] for p in per]

    def _concat_per_record(self, wires, keys, strict, out_dtypes, device, out, string_columns=False):
        return self._per_record(wires, keys, strict, out_dtypes, device, out,
                                lambda k, parts: "zero-dimensional arrays cannot be concatenated" if any(a.ndim == 0 for a in parts) else None,
                                lambda k, parts: np.concatenate(parts, axis=0),
                                (lambda k, parts: self._string_column(k, parts, device, out)) if string_columns else None)

    def _string_column(self, key, parts, device: bool, out) -> BytesColumn:
        """The per-response route's BytesColumn of one string output, with the concatenation's errors (ValueError: rank 0, another
        dtype, another rank or other trailing dims)."""
        if key in out:
            raise ValueError(f"output {key!r}: out= does not take string columns")
        if any(isinstance(a, _RawStrings) and len(a.shape) == 0 or not isinstance(a, _RawStrings) and a.ndim == 0 for a in parts):
            raise ValueError("zero-dimensional arrays cannot be concatenated")
        if not all(isinstance(a, _RawStrings) for a in parts):
            raise ValueError(f"output {key!r}: responses disagree on the dtype")
        if len({a.shape[1:] for a in parts}) > 1 or len({len(a.shape) for a in parts}) > 1:
            raise ValueError(f"output {key!r}: all the input array dimensions except for the concatenation axis must match exactly")
        return self._bytes_column([b for a in parts for b in a.strings], (sum(a.shape[0] for a in parts),) + tuple(parts[0].shape[1:]),
                                  device)

    def _bytes_column(self, strs, shape, device: bool) -> BytesColumn:
        offsets = np.zeros(len(strs) + 1, np.int64)
        np.cumsum(np.fromiter(map(len, strs), np.int64, len(strs)), out=offsets[1:])
        data = np.frombuffer(b"".join(strs), np.uint8)
        if device:
            return BytesColumn(self.device_array(data), self.device_array(offsets), shape)
        return BytesColumn(data.copy(), offsets, shape)

    def _concat_deliver(self, key, arr: np.ndarray, device: bool, out):
        dst = out.get(key)
        if dst is None:
            return self.device_array(arr) if device else arr
        view = _check_out(key, dst, arr.dtype, arr.shape)
        if view is None:
            np.copyto(dst, arr)
        elif arr.nbytes:
            a = np.ascontiguousarray(arr)
            N.check(self._lib.b200tfs_memcpy_h2d(self._ctx, view[0], a.ctypes.data, a.nbytes))
            self.sync()
        return dst

    def _key_device(self, native, wires, buf, off, ln, keys, strict, out_dtypes, out, shape_of, place,
                    strings: bool = False) -> Optional["_KeyLaunch"]:
        """A per-key device route up to the results of its decode, or None when the batch holds a case it leaves to the
        per-response route.  `native`: the route's key struct and its layout, decode and results entry points.  The host layout
        runs first, so nothing is written into `out` for a batch the route then refuses.  `shape_of(i, key struct, numpy type)`
        is key i's result shape (None: refused); `place(key structs, pointers, shapes, numpy types)` completes the key structs
        once the destinations are known (False: refused).  `strings`: DT_STRING keys are the route's too (their destination is
        int64 offsets, which `shape_of` sizes), except that `out` may not name one (ValueError)."""
        if len(keys) > N.CONCAT_MAX_KEYS:
            return None
        key_type, layout, decode, results = native
        n, nk = len(wires), len(keys)
        kb = [k.encode("utf-8") for k in keys]
        cast_code = 0
        if out_dtypes:
            cast_code = None if strict else _narrowing_cast(out_dtypes)
            if cast_code is None:
                return None
        ks = (key_type * nk)()
        for i, k in enumerate(kb):
            ks[i].key, ks[i].key_len = k, len(k)
        N.check(layout(buf.ctypes.data, n, off, ln, nk, ks, cast_code))
        shapes, np_types = [], []
        for i in range(nk):
            c = ks[i]
            if c.status != N.OK or c.dtype == DT_STRING and not strings or strict and c.dtype in (DT_BFLOAT16, DT_COMPLEX64, DT_COMPLEX128):
                return None
            if c.dtype == DT_STRING and keys[i] in out:
                raise ValueError(f"output {keys[i]!r}: out= does not take string columns")
            if cast_code and not _narrowing_fits(c.dtype, keys[i], out_dtypes):
                return None
            if c.dtype == DT_STRING:
                np_types.append(np.dtype(np.int64))
            else:
                np_types.append(np.dtype(numpy_for_enum(cast_code if cast_code and c.dtype == DT_FLOAT else int(c.dtype))))
            shape = shape_of(i, c, np_types[i])
            if shape is None:
                return None
            shapes.append(shape)
        dev, ptrs, holds = self._key_destinations(keys, out, shapes, np_types)
        if not place(ks, ptrs, shapes, np_types):
            return None
        wire = D.DeviceArray(self, (len(buf),), np.uint8).copy_from_host(buf)
        with self._decode_modes(cast_code):
            N.check(decode(self._ctx, wire.ptr, n, off, ln, nk, ks))
        outs, specs, rec_status = (N.Output * (n * nk))(), (N.ModelSpec * n)(), (C.c_int32 * n)()
        N.check(results(self._ctx, n, nk, outs, specs, rec_status))   # synchronises
        return _KeyLaunch(ks, wire, outs, rec_status, [self._spec(buf, int(off[r]), specs[r]) for r in range(n)],
                          shapes, np_types, dev, ptrs, holds)

    def _concat_device(self, wires, buf, off, ln, keys, strict, out_dtypes, device, out, string_columns=False):
        """The device route (b200tfs_decode_concat): parse, one-CTA plan, move, varint decode - or None when the batch holds
        a case it leaves to the per-response route.  `string_columns`: with b200tfs_concat_strings entries (string index, scan,
        copy and fix kernels) when a requested key is DT_STRING."""
        nk = len(keys)
        sc = (N.ConcatStrings * nk)() if string_columns else None
        data = {}
        lib = self._lib

        def has_strings(ck):
            return any(ck[i].dtype == DT_STRING and ck[i].status == N.OK for i in range(nk))

        def place(ck, ptrs, shapes, np_types):
            for i in range(nk):
                ck[i].dst, ck[i].dst_cap = ptrs[i], int(ck[i].bytes)
                if ck[i].dtype == DT_STRING:
                    data[i] = D.DeviceArray(self, (int(sc[i].data_bytes),), np.uint8)
                    sc[i].data, sc[i].data_cap = data[i].ptr, int(sc[i].data_bytes)
            return True
        if string_columns:
            native = (N.ConcatKey, lambda *a: lib.b200tfs_concat_strings_layout(*a[:6], sc, a[6]),
                      lambda *a: lib.b200tfs_decode_concat_strings(*a, sc if has_strings(a[6]) else None), lib.b200tfs_concat_results)
        else:
            native = (N.ConcatKey, lib.b200tfs_concat_layout, lib.b200tfs_decode_concat, lib.b200tfs_concat_results)
        f = self._key_device(native, wires, buf, off, ln, keys, strict, out_dtypes, out,
                             lambda i, c, np_type: (int(sc[i].strings) + 1,) if c.dtype == DT_STRING else tuple(int(c.dims[d]) for d in range(c.rank)),
                             place, strings=string_columns)
        if f is None:
            return None
        n = len(wires)
        if any(f.outs[r * nk + i].status != N.OK for i in data for r in range(n)):
            return None       # E_NONCANONICAL (a TensorProto in several `value` occurrences): the per-response route
        raw = np.frombuffer(f.outs, dtype=np.uint8).reshape(n * nk, C.sizeof(N.Output))
        status = raw[:, N.Output.status.offset: N.Output.status.offset + 4].copy().view(np.int32).ravel()
        redo = set(np.flatnonzero(status != N.OK).tolist())
        if strict:     # the reference reads half_val as VALUES; the device wrote TF's bit patterns
            for i in range(nk):
                if f.keys[i].dtype == DT_HALF:
                    redo.update(r * nk + i for r in range(n))
        jobs = []
        for j in sorted(redo):
            r, i = divmod(j, nk)
            o = f.outs[j]
            if f.rec_status[r] != N.OK or not _to_unpack(o, N.E_NONCANONICAL):
                return None
            _, dst_code, _ = self._resolve_output(o, strict, out_dtypes.get(keys[i]) if out_dtypes else None)
            if o.n_elems:
                jobs.append((j, r, f.ptrs[i] + int(o.dst_off), dst_code))
        if jobs:
            m = len(jobs)
            o_arr = (N.Output * m)(*[f.outs[j[0]] for j in jobs])
            rec = (C.c_uint64 * m)(*[int(off[j[1]]) for j in jobs])
            dd = (C.c_void_p * m)(*[j[2] for j in jobs])
            codes = (C.c_int32 * m)(*[j[3] for j in jobs])
            st = (C.c_int32 * m)()
            N.check(self._lib.b200tfs_unpack_outputs(self._ctx, f.wire.ptr, m, o_arr, rec, dd, codes, st))
            if any(st[q] != N.OK for q in range(m)):
                return None
        result = self._key_deliver(keys, out, device, f.shapes, f.np_types, f.dev, f.ptrs)
        for i, a in data.items():
            c = f.keys[i]
            shape = tuple(int(c.dims[d]) for d in range(c.rank))
            result[keys[i]] = BytesColumn(a if device else a.copy_to_host(), result[keys[i]], shape)
        self.concat_device_calls += 1
        return result, f.specs

    def _key_destinations(self, keys, out, shapes, np_types):
        """Device destinations of a per-key device decode: the caller's device arrays, else device arrays of our own (returned,
        or copied into the host result).  Returns (arrays, pointers, keep-alives)."""
        dev, ptrs, holds = [], [], []
        for i, k in enumerate(keys):
            dst = out.get(k)
            view = None if dst is None else _check_out(k, dst, np_types[i], shapes[i], contiguous=True)
            if view is not None:
                dev.append(dst)
                ptrs.append(view[0])
                holds.append(view)
            else:
                a = D.DeviceArray(self, shapes[i], np_types[i])
                dev.append(a)
                ptrs.append(a.ptr)
        return dev, ptrs, holds

    def _key_deliver(self, keys, out, device, shapes, np_types, dev, ptrs):
        """{key: result} of a per-key device decode that finished: the caller's device array, the caller's host array or a new
        one (one device-to-host copy each), or our device array.  Synchronises."""
        result = {}
        for i, k in enumerate(keys):
            dst = out.get(k)
            if dst is not None and D.is_device_object(dst):
                result[k] = dst
            elif dst is not None or not device:
                host = dst if dst is not None else np.empty(shapes[i], dtype=np_types[i])
                if host.nbytes:
                    N.check(self._lib.b200tfs_memcpy_d2h(self._ctx, host.ctypes.data, ptrs[i], host.nbytes))
                result[k] = host
            else:
                result[k] = dev[i]
        self.sync()
        return result

    # ---- batch decode into one padded tensor per key -----------------------------------------------------
    def decode_predict_responses_padded(self, wires: Sequence[bytes], keys: Optional[Sequence[str]] = None, *, pad_value=0,
                                        pad_to: Optional[Mapping] = None, strict: bool = False, out_dtypes: Optional[Mapping] = None,
                                        device: bool = False, out: Optional[Mapping] = None, string_columns: bool = False,
                                        string_pad: bytes = b""
                                        ) -> Tuple[Dict[str, object], Dict[str, np.ndarray], List[DecodedSpec]]:
        """Decode a batch of PredictResponses with ragged trailing dimensions into ONE padded tensor per output - what
        ``pad_sequence`` / ``tf.keras.utils.pad_sequences`` give: for every key, the rows of all responses concatenated along axis
        0, every other axis padded at its end with ``pad_value`` to the batch maximum, or to ``pad_to[key]`` (the trailing dims).
        Bit for bit, and with the same exceptions, what this does with the per-response decode::

            parts = [decode_predict_responses([w], strict=strict, out_dtypes=out_dtypes)[0][0][key] for w in wires]
            tail = pad_to[key] if key in pad_to else elementwise max of p.shape[1:]     # rank 0 / other ranks: ValueError
            res = np.full((sum(p.shape[0] for p in parts), *tail), pad_value, dtype)    # other dtypes: ValueError
            # part r fills res[r0:r0 + rows_r, :d1, :d2, ...]; a part larger than pad_to: ValueError

        ``keys``, ``strict``, ``out_dtypes``, ``device`` and ``out`` as for ``decode_predict_responses_concat`` (a narrowed output
        gets the pad converted to the narrowed dtype).  Returns ``({key: tensor}, {key: int64[n, rank] shape of every response's
        output}, [DecodedSpec per response])``.

        ``string_columns=True``: every DT_STRING output comes back as a padded ``BytesColumn`` of shape ``(rows, *tail)`` - in C
        order, each position inside a response's own dims holds that response's raw ``string_val`` bytes (no UTF-8 check, NULs
        and high bytes kept) and every other position of its rows holds ``string_pad`` (``bytes``) - with ``offsets`` int64[m + 1]
        from 0, decoded on the device in the same call as the numeric outputs (``DeviceArray`` data and offsets with
        ``device=True``, numpy arrays otherwise), with the errors above.  The column and the shapes table feed
        ``encode_predict_requests_padded`` directly.  ``out`` naming a string output raises ValueError.  Without it, string
        outputs are decoded on the host into numpy str arrays (and ``device=True`` raises TypeError for them).
        """
        buf, off, ln, keys, out_dtypes, out = self._requested(wires, keys, out, out_dtypes, "need at least one response to pad")
        pad_to = dict(pad_to or {})
        string_pad = bytes(string_pad)
        fast = self._padded_device(wires, buf, off, ln, keys, pad_value, pad_to, strict, out_dtypes, device, out, string_columns,
                                   string_pad)
        if fast is not None:
            return fast
        return self._padded_per_record(wires, keys, pad_value, pad_to, strict, out_dtypes, device, out, string_columns, string_pad)

    @staticmethod
    def _padded_tail(k, pad_to, rank: int, dims) -> Tuple[int, ...]:
        """The trailing dims of key k's padded tensor: pad_to[k], else the elementwise maximum of the parts' `dims` (ValueError:
        pad_to of another rank)."""
        tail = tuple(int(x) for x in pad_to[k]) if k in pad_to else tuple(max(s[d] for s in dims) for d in range(1, rank))
        if len(tail) != rank - 1:
            raise ValueError(f"output {k!r}: pad_to has {len(tail)} trailing dims, the output {rank - 1}")
        return tail

    @staticmethod
    def _padded_fits(k, tail, shape) -> None:
        if any(shape[d] > tail[d - 1] for d in range(1, len(shape))):
            raise ValueError(f"output {k!r}: a response of shape {shape} does not fit pad_to {tail}")

    def _padded_per_record(self, wires, keys, pad_value, pad_to, strict, out_dtypes, device, out, string_columns=False, string_pad=b""):
        shapes = {}

        def bad_rank(k, parts):
            rank = parts[0].ndim
            if rank == 0 or any(a.ndim != rank for a in parts):
                return f"output {k!r}: every response must have the same rank >= 1 to be padded"
            return None

        def pad(k, parts):
            rank = parts[0].ndim
            tail = self._padded_tail(k, pad_to, rank, [a.shape for a in parts])
            res = np.full((sum(a.shape[0] for a in parts), *tail), pad_value, parts[0].dtype)
            r0 = 0
            for a in parts:
                self._padded_fits(k, tail, a.shape)
                res[(slice(r0, r0 + a.shape[0]),) + tuple(slice(0, d) for d in a.shape[1:])] = a
                r0 += a.shape[0]
            shapes[k] = np.array([a.shape for a in parts], dtype=np.int64).reshape(len(parts), rank)
            return res

        def string_column(k, parts):
            """The padded BytesColumn of string output k, with the padded decode's errors."""
            if k in out:
                raise ValueError(f"output {k!r}: out= does not take string columns")
            if not all(isinstance(a, _RawStrings) for a in parts):
                raise ValueError(f"output {k!r}: responses disagree on the dtype")
            rank = len(parts[0].shape)
            if rank == 0 or any(len(a.shape) != rank for a in parts):
                raise ValueError(f"output {k!r}: every response must have the same rank >= 1 to be padded")
            tail = self._padded_tail(k, pad_to, rank, [a.shape for a in parts])
            res = np.empty((sum(a.shape[0] for a in parts), *tail), object)
            res.fill(string_pad)
            r0 = 0
            for a in parts:
                self._padded_fits(k, tail, a.shape)
                own = np.empty(len(a.strings), object)
                own[:] = a.strings
                res[(slice(r0, r0 + a.shape[0]),) + tuple(slice(0, d) for d in a.shape[1:])] = own.reshape(a.shape)
                r0 += a.shape[0]
            shapes[k] = np.array([a.shape for a in parts], dtype=np.int64).reshape(len(parts), rank)
            return self._bytes_column(res.ravel().tolist(), res.shape, device)
        result, specs = self._per_record(wires, keys, strict, out_dtypes, device, out, bad_rank, pad,
                                         string_column if string_columns else None)
        return result, shapes, specs

    def _padded_device(self, wires, buf, off, ln, keys, pad_value, pad_to, strict, out_dtypes, device, out, string_columns=False,
                       string_pad=b""):
        """The device route (b200tfs_decode_padded): parse, one-CTA plan, destination-major emit, varint decode - or None
        when the batch holds a case it leaves to the response-by-response route.  `string_columns`: with b200tfs_padded_strings
        entries (string index, scan, copy and fix kernels) when a requested key is DT_STRING."""
        nk = len(keys)
        pads, columns, data = [], {}, {}
        ps = (N.PaddedStrings * nk)() if string_columns else None
        lib = self._lib

        def shape_of(i, c, np_type):
            if strict and c.dtype == DT_HALF:
                return None   # the reference reads half_val as values, the device writes TF's bit patterns
            tail = tuple(int(c.dims[d]) for d in range(1, c.rank))
            if keys[i] in pad_to:
                want = tuple(int(x) for x in pad_to[keys[i]])
                if len(want) != len(tail) or any(t > w for t, w in zip(tail, want)):
                    return None   # the definition raises, after decoding every response
                tail = want
            if c.dtype == DT_STRING:   # its destination is the column's int64 offsets
                columns[i] = (int(c.dims[0]),) + tail
                pads.append(b"")
                return (int(np.prod(columns[i], dtype=np.int64)) + 1,)
            try:
                pads.append(np.full((1,), pad_value, np_type).tobytes())
            except Exception:     # noqa: BLE001 - the definition raises it, after decoding every response
                return None
            return (int(c.dims[0]),) + tail

        def place(pk, ptrs, shapes, np_types):
            if any(p % 16 for p in ptrs):
                return False      # the emit writes whole 16-byte vectors
            for i in range(nk):
                shape = columns.get(i, shapes[i])
                pk[i].dst, pk[i].dst_cap, pk[i].rank = ptrs[i], int(np.prod(shapes[i], dtype=np.int64)) * np_types[i].itemsize, len(shape)
                for d in range(1, len(shape)):
                    pk[i].dims[d] = shape[d]
                C.memmove(pk[i].pad_bits, pads[i], len(pads[i]))
                if i in columns:
                    m = shapes[i][0] - 1
                    cap = int(ps[i].data_bytes) + (m - int(ps[i].strings)) * len(string_pad)
                    data[i] = D.DeviceArray(self, (cap,), np.uint8)
                    ps[i].data, ps[i].data_cap, ps[i].pad, ps[i].pad_len = data[i].ptr, cap, C.cast(C.c_char_p(string_pad), C.c_void_p), len(string_pad)
            return True
        if string_columns:
            native = (N.PadKey, lambda *a: lib.b200tfs_padded_strings_layout(*a[:6], ps, a[6]),
                      lambda *a: lib.b200tfs_decode_padded_strings(*a, ps if columns else None), lib.b200tfs_padded_results)
        else:
            native = (N.PadKey, lib.b200tfs_padded_layout, lib.b200tfs_decode_padded, lib.b200tfs_padded_results)
        f = self._key_device(native, wires, buf, off, ln, keys, strict, out_dtypes, out, shape_of, place, strings=string_columns)
        if f is None:
            return None
        n = len(wires)
        if any(f.rec_status[r] != N.OK for r in range(n)) or any(f.outs[j].status != N.OK for j in range(n * nk)):
            return None
        ranks = [len(columns.get(i, f.shapes[i])) for i in range(nk)]
        rec_shapes = {k: np.array([list(f.outs[r * nk + i].dims)[: ranks[i]] for r in range(n)], dtype=np.int64).reshape(n, ranks[i])
                      for i, k in enumerate(keys)}
        result = self._key_deliver(keys, out, device, f.shapes, f.np_types, f.dev, f.ptrs)
        for i, a in data.items():
            result[keys[i]] = BytesColumn(a if device else a.copy_to_host(), result[keys[i]], columns[i])
        self.padded_device_calls += 1
        return result, rec_shapes, f.specs

    # ---- Classify / Regress responses ------------------------------------------------------------------
    def decode_regression_responses(self, wires: Sequence[bytes], *, device: bool = False, out=None) -> RegressionBatch:
        """Decode a batch of RegressionResponses into one float32 array of every regression's value, response after response -
        ``np.array([r.value for w in wires for r in RegressionResponse.FromString(w).result.regressions], np.float32)`` bit
        for bit, raising what FromString raises.  ``device=True``: ``values`` is a ``DeviceArray`` (of the used rows);
        ``out=``: a C-contiguous float32 device array or numpy / ``pinned_empty`` array of at least ``rows`` elements, of
        which ``out[:rows]`` is returned (nothing is written into it when the call raises)."""
        return self._decode_example_responses(N.RESP_REGRESS, wires, device, out)

    def decode_classification_responses(self, wires: Sequence[bytes], *, device: bool = False, out=None) -> ClassificationBatch:
        """Decode a batch of ClassificationResponses into one float32 ``[rows, C]`` array of scores - ``np.array([[c.score for c
        in cl.classes] for w in wires for cl in ClassificationResponse.FromString(w).result.classifications], np.float32)``
        bit for bit - raising what FromString raises, and ValueError when the examples disagree on the number of classes C.
        ``device`` and ``out`` (at least ``rows`` rows of C columns) as for ``decode_regression_responses``."""
        return self._decode_example_responses(N.RESP_CLASSIFY, wires, device, out)

    def _xr_buffers(self, values: int, labels: int):
        """The codec's own device destinations, grown to hold `values` floats and `labels` label references."""
        have = self._xr_scratch
        if have is None or have[0].nbytes < 4 * values or have[1].nbytes < C.sizeof(N.LabelRef) * labels:
            v = max(values, have[0].nbytes // 4 if have else 0)
            lab = max(labels, have[1].nbytes // C.sizeof(N.LabelRef) if have else 0)
            self._xr_scratch = have = (D.DeviceArray(self, (max(v, 1),), np.float32), D.DeviceArray(self, (max(lab, 1), 2), np.uint32))
        return have

    def _decode_example_responses(self, kind, wires, device, out):
        n = len(wires)
        cls = kind == N.RESP_CLASSIFY
        if n == 0:
            return self._example_batch_host(kind, wires, device, out)
        buf, off, ln = self._pack_wires(wires)
        max_rows, max_values = C.c_uint64(), C.c_uint64()
        N.check(self._lib.b200tfs_example_response_bound(kind, n, ln, C.byref(max_rows), C.byref(max_values)))
        mv = int(max_values.value)
        # the kernels write the codec's scratch; the result reaches the caller's destination only once the batch has decoded
        scratch_v, scratch_l = self._xr_buffers(mv, mv if cls else 0)
        vptr, lptr, lcap = scratch_v.ptr, (scratch_l.ptr if cls else None), (mv if cls else 0)
        N.check(self._lib.b200tfs_decode_example_responses_host_async(self._ctx, kind, buf.ctypes.data, n, off, ln, vptr, mv, lptr, lcap))
        per, specs, batch = (C.c_int64 * (3 * n))(), (N.ModelSpec * n)(), (C.c_int64 * 5)()
        N.check(self._lib.b200tfs_example_response_results(self._ctx, n, per, specs, batch))   # synchronises
        if int(batch[3]) != N.OK:      # a response the device route does not decode: the definition itself, response by response
            return self._example_batch_host(kind, wires, device, out)
        res = self._xr_deliver(cls, buf, off, n, per, specs, batch, vptr, lptr, device, out)
        self.example_response_device_calls += 1
        return res

    def _xr_deliver(self, cls, buf, off, n, per, specs, batch, vptr, lptr, device, out):
        """The batch one task of a device decode left: `per`, `specs` and `batch` as b200tfs_example_response_results gives them,
        its values at vptr and (cls) its label references at lptr on the device."""
        rows, ncls, same = int(batch[0]), int(batch[1]), bool(batch[2])
        counts = np.array([per[3 * i + 1] for i in range(n)], dtype=np.int64)
        spec_list = [self._spec(buf, int(off[i]), specs[i]) for i in range(n)]
        vals = self._example_out((rows, ncls) if cls else (rows,), device, out, src_dev=vptr)
        if cls:
            nref = ncls if same else rows * ncls
            refs = np.empty((nref, 2), np.uint32)
            if nref:
                N.check(self._lib.b200tfs_memcpy_d2h(self._ctx, refs.ctypes.data, lptr, refs.nbytes))
        self.sync()
        if not cls:
            return RegressionBatch(vals, counts, spec_list)
        row_of = np.repeat(np.arange(n), counts)
        text = lambda i, k: self._text(buf, int(off[row_of[i]]) + int(refs[i * ncls + k, 0]), int(refs[i * ncls + k, 1]))   # noqa: E731
        if same:
            class_labels = [text(0, k) for k in range(ncls)] if rows else []
            return ClassificationBatch(vals, counts, spec_list, class_labels, lambda: [class_labels] * rows)
        return ClassificationBatch(vals, counts, spec_list, None, lambda: [[text(i, k) for k in range(ncls)] for i in range(rows)])

    def _example_out(self, shape, device, out, src_dev=None, host=None):
        """The decoded float32 array of `shape` - on the device at src_dev, or the host array `host` - delivered where the caller
        asked: into ``out`` (``out[:rows]`` is returned; a device array that cannot be sliced must have exactly `rows` rows), a new
        ``DeviceArray`` (device=True) or a new numpy array.  ``out`` is checked before anything is written into it."""
        rows, nbytes = shape[0], 4 * int(np.prod(shape, dtype=np.int64))
        if out is not None and D.is_device_object(out):
            ptr, oshape, odtype, hold = D.device_view(out)
            sliceable = hasattr(out, "__getitem__")
            if odtype != np.float32 or len(oshape) != len(shape) or tuple(oshape[1:]) != tuple(shape[1:]) or oshape[0] < rows \
                    or (not sliceable and oshape[0] != rows):
                raise ValueError(f"out: {odtype}{tuple(oshape)} cannot take {tuple(shape)} float32 values"
                                 + ("" if sliceable else " (an array that cannot be sliced must have exactly that shape)"))
            dst = out
        elif device and out is None:
            dst = D.DeviceArray(self, shape, np.float32)
            ptr = dst.ptr
        else:
            if out is not None and (not isinstance(out, np.ndarray) or out.dtype != np.float32 or not out.flags.c_contiguous
                                    or out.ndim != len(shape) or out.shape[1:] != tuple(shape[1:]) or len(out) < rows):
                raise ValueError(f"out must be a C-contiguous float32 array of at least {tuple(shape)} (rows first)")
            arr = np.empty(shape, np.float32) if out is None else out[:rows]
            if host is not None:
                arr[...] = host
            elif nbytes:
                N.check(self._lib.b200tfs_memcpy_d2h(self._ctx, arr.ctypes.data, src_dev, nbytes))
                self.sync()
            return arr
        if nbytes:
            if host is not None:
                a = np.ascontiguousarray(host, dtype=np.float32)
                N.check(self._lib.b200tfs_memcpy_h2d(self._ctx, ptr, a.ctypes.data, nbytes))
            else:
                N.check(self._lib.b200tfs_memcpy_d2d(self._ctx, ptr, src_dev, nbytes))
            self.sync()
        return dst[:rows] if dst is out and hasattr(out, "__getitem__") else dst

    def _example_batch_host(self, kind, wires, device, out):
        """The definition, response by response, with protobuf on the host: what the device route hands over when a response
        does not decode there (malformed, ragged class counts, rows past the caller's ``out``)."""
        from tensorflow_serving.apis.classification_pb2 import ClassificationResponse
        from tensorflow_serving.apis.regression_pb2 import RegressionResponse

        cls = kind == N.RESP_CLASSIFY
        msgs = [(ClassificationResponse if cls else RegressionResponse).FromString(bytes(w)) for w in wires]
        return self._example_batch_of(cls, [m.result for m in msgs], [m.model_spec for m in msgs], device, out)

    def _example_batch_of(self, cls, results, model_specs, device, out):
        """The batch of parsed ClassificationResults (cls) or RegressionResults and their model_specs, one of each per response."""
        specs = [DecodedSpec(s.name, s.version.value, s.HasField("version"), s.version_label, s.signature_name) for s in model_specs]
        if cls:
            rows = [cl.classes for m in results for cl in m.classifications]
            if len({len(r) for r in rows}) > 1:
                raise ValueError("examples disagree on the number of classes")
            ncls = len(rows[0]) if rows else 0
            vals = np.array([[c.score for c in r] for r in rows], np.float32).reshape(len(rows), ncls)
            counts = np.array([len(m.classifications) for m in results], dtype=np.int64)
            labels = [[c.label for c in r] for r in rows]
        else:
            vals = np.array([r.value for m in results for r in m.regressions], np.float32)
            counts = np.array([len(m.regressions) for m in results], dtype=np.int64)
        res = self._example_out(vals.shape, device, out, host=vals)
        if not cls:
            return RegressionBatch(res, counts, specs)
        same = all(r == labels[0] for r in labels)
        return ClassificationBatch(res, counts, specs, list(labels[0]) if same and labels else ([] if same else None), labels)

    # ---- MultiInference responses -----------------------------------------------------------------
    def decode_multi_inference_responses(self, wires: Sequence[bytes], methods: Sequence[str], *, device: bool = False,
                                         out=None) -> List[Union[ClassificationBatch, RegressionBatch]]:
        """Decode a batch of MultiInferenceResponses of a request whose tasks have the method names ``methods``
        (``CLASSIFY_METHOD_NAME`` / ``REGRESS_METHOD_NAME``, in task order): one ``ClassificationBatch`` or ``RegressionBatch``
        per task, in task order.  Task t's batch is what ``decode_classification_responses`` / ``decode_regression_responses``
        give for ``results[t]`` of every response, its specs each result's own model_spec.  Raises what
        ``MultiInferenceResponse.FromString`` raises, and ValueError when a response has another number of results than
        ``methods``, when a result is not the one its method names (an empty one included), or when a classify task's examples
        disagree on the number of classes.  ``device`` as there; ``out`` is None or a sequence parallel to ``methods`` whose
        entries (None: a new array) follow the rules of ``out`` there."""
        kinds = [_method_kind(m) for m in methods]
        T = len(kinds)
        if not T:
            raise ValueError("a MultiInference decode needs at least one task")
        outs = [None] * T if out is None else list(out)
        if len(outs) != T:
            raise ValueError(f"out has {len(outs)} entries for {T} tasks")
        n = len(wires)
        if n == 0:
            return self._multi_batch_host(kinds, wires, device, outs)
        buf, off, ln = self._pack_wires(wires)
        kv = (C.c_int32 * T)(*kinds)
        max_rows, max_values = (C.c_uint64 * T)(), (C.c_uint64 * T)()
        N.check(self._lib.b200tfs_multi_inference_response_bound(T, kv, n, ln, max_rows, max_values))
        mv = int(max_values[0])           # every task has the same bound
        cls_of = [k == N.RESP_CLASSIFY for k in kinds]
        label_at = list(np.cumsum([0] + cls_of[:-1]))     # the classify tasks' places in the label scratch
        scratch_v, scratch_l = self._xr_buffers(T * mv, sum(cls_of) * mv)
        vptrs = [scratch_v.ptr + 4 * mv * t for t in range(T)]
        lptrs = [scratch_l.ptr + C.sizeof(N.LabelRef) * mv * int(label_at[t]) if cls_of[t] else None for t in range(T)]
        caps = (C.c_uint64 * T)(*[mv] * T)
        lcaps = (C.c_uint64 * T)(*[mv if c else 0 for c in cls_of])
        N.check(self._lib.b200tfs_decode_multi_inference_responses_host_async(self._ctx, T, kv, buf.ctypes.data, n, off, ln,
                                                                              (C.c_void_p * T)(*vptrs), caps, (C.c_void_p * T)(*lptrs),
                                                                              lcaps))
        per, specs, batch = (C.c_int64 * (3 * n * T))(), (N.ModelSpec * (n * T))(), (C.c_int64 * (5 * T))()
        N.check(self._lib.b200tfs_multi_inference_response_results(self._ctx, n, T, per, specs, batch))   # synchronises
        if any(int(batch[5 * t + 3]) != N.OK for t in range(T)):   # the definition itself, response by response
            return self._multi_batch_host(kinds, wires, device, outs)
        res = [self._xr_deliver(cls_of[t], buf, off, n, per[3 * n * t: 3 * n * (t + 1)], specs[n * t: n * (t + 1)],
                                batch[5 * t: 5 * (t + 1)], vptrs[t], lptrs[t], device, outs[t]) for t in range(T)]
        self.multi_inference_device_calls += 1
        return res

    def _multi_batch_host(self, kinds, wires, device, outs):
        """The definition of ``decode_multi_inference_responses`` with protobuf on the host: what the device route hands over when
        a response does not decode there."""
        from tensorflow_serving.apis.inference_pb2 import MultiInferenceResponse

        msgs = [MultiInferenceResponse.FromString(bytes(w)) for w in wires]
        T = len(kinds)
        for i, m in enumerate(msgs):
            if len(m.results) != T:
                raise ValueError(f"response {i} has {len(m.results)} results for {T} tasks")
            for t, k in enumerate(kinds):
                want = "classification_result" if k == N.RESP_CLASSIFY else "regression_result"
                if m.results[t].WhichOneof("result") != want:
                    raise ValueError(f"response {i}: result {t} is {m.results[t].WhichOneof('result')}, its task wants {want}")
        res = []
        for t, k in enumerate(kinds):
            cls = k == N.RESP_CLASSIFY
            body = [m.results[t].classification_result if cls else m.results[t].regression_result for m in msgs]
            res.append(self._example_batch_of(cls, body, [m.results[t].model_spec for m in msgs], device, outs[t]))
        return res

    @staticmethod
    def _decode_strings(buf: np.ndarray, base: int, o: N.Output, rec_len: int = 0, key: str = "") -> np.ndarray:
        proto = Codec._string_proto(buf, base, o, rec_len, key)
        shape = tuple(int(d.size) for d in proto.tensor_shape.dim)     # the host message is at hand: any rank
        return np.array([e for e in proto.string_val], dtype=np.str_).reshape(*shape)

    @staticmethod
    def _string_proto(buf: np.ndarray, base: int, o: N.Output, rec_len: int = 0, key: str = ""):
        """The TensorProto of a string output, as the runtime merges it."""
        from tensorflow.core.framework.tensor_pb2 import TensorProto

        proto = TensorProto.FromString(buf[base + o.msg_off: base + o.msg_off + o.msg_len].tobytes())
        if rec_len and (len(proto.string_val) != o.n_strings or len(proto.tensor_shape.dim) != o.rank):
            # the map entry carried its TensorProto in several `value` occurrences, which the runtime merges (the table counts
            # all of them; msg_off is the last one): parse the whole response the way the runtime does
            from tensorflow_serving.apis.predict_pb2 import PredictResponse

            proto = PredictResponse.FromString(buf[base: base + rec_len].tobytes()).outputs[key]
        return proto

    def decode_predict_response(self, wire: bytes, *, out: Optional[Mapping[str, np.ndarray]] = None, **kw) -> Tuple[Dict[str, np.ndarray], DecodedSpec]:
        """One response.  ``out={key: array}``: the named outputs are written into the caller's arrays (dtype and shape must
        match); when the response has that one fixed-width output and the array came from ``pinned_empty``, the device-to-host
        copy lands in it directly (no staging buffer, no extra copy on the host)."""
        if out:
            direct = self._decode_into_pinned(wire, out, kw.get("strict", False)) if len(out) == 1 and not kw.get("out_dtypes") else None
            if direct is not None:
                return direct
            arrays, spec = self.decode_predict_responses([wire], **kw)[0]
            for k, dst in out.items():
                if k not in arrays:
                    raise KeyError(k)
                _check_out(k, dst, arrays[k].dtype, arrays[k].shape)
                np.copyto(dst, arrays[k])
                arrays[k] = dst
            return arrays, spec
        return self.decode_predict_responses([wire], **kw)[0]

    def _decode_into_pinned(self, wire, out: Mapping[str, np.ndarray], strict: bool):
        (key, arr), = out.items()
        cap = self._pinned.capacity(arr)
        if cap is None or not len(wire):
            return None
        launch = self._fused_launch([wire], dst=arr, stride=cap & ~255)
        if launch is None or len(launch.tables[0]) != 1:
            return None                                  # not the single-output case after all: the general path redoes it
        o = launch.tables[0].get(key)
        if o is None or not _stored(o) or o.dst_off != 0:
            return None
        np_type, dst_code, shape = self._resolve_output(o, strict, None)
        if not _stored_as(o, dst_code) or np.dtype(np_type) != arr.dtype or tuple(shape) != arr.shape:
            return None
        return {key: arr}, self._spec(launch.buf, 0, launch.specs[0])

    def decode_tensor_protos(self, wires: Sequence[bytes], *, strict: bool = False, out_dtype=None) -> List[np.ndarray]:
        """``tensor_proto_to_ndarray`` for serialised TensorProto messages."""
        n = len(wires)
        if n == 0:
            return []
        buf, off, ln = self._pack_wires(wires)
        outs = (N.Output * n)()
        status = (C.c_int32 * n)()
        N.check(self._lib.b200tfs_parse_tensor_protos_host(self._ctx, buf.ctypes.data, n, off, ln, outs, status))
        results: List[Optional[np.ndarray]] = [None] * n
        jobs = []
        for i in range(n):
            N.check(status[i])
            o = outs[i]
            if int(o.dtype) == DT_STRING and o.status == N.OK:
                results[i] = self._decode_strings(buf, int(off[i]), o)
                continue
            np_type, dst_code, shape = self._resolve_output(o, strict, out_dtype)
            jobs.append((results, i, o, np_type, dst_code, shape, int(off[i])))
        self._unpack_to_host(jobs)
        return results  # type: ignore[return-value]


# ---- zero-copy helpers -----------------------------------------------------------------------------
# CPython only: PyBytes_FromStringAndSize(NULL, n) is the documented way to make a bytes object whose buffer the caller
# fills before anyone else sees the object (https://docs.python.org/3/c-api/bytes.html).  The object is not hashed,
# interned or shared until the library has written every byte of it; other interpreters take the copying path.
import platform as _platform

_HAVE_NEW_BYTES = _platform.python_implementation() == "CPython" and hasattr(C, "pythonapi")
if _HAVE_NEW_BYTES:
    _PyBytes_FromStringAndSize = C.pythonapi.PyBytes_FromStringAndSize
    _PyBytes_FromStringAndSize.restype = C.py_object
    _PyBytes_FromStringAndSize.argtypes = [C.c_void_p, C.c_ssize_t]
    _PyBytes_AsString = C.pythonapi.PyBytes_AsString
    _PyBytes_AsString.restype = C.c_void_p
    _PyBytes_AsString.argtypes = [C.py_object]


def _new_bytes(n: int):
    """An uninitialised bytes object of n bytes and the address of its buffer: the device-to-host copy lands
    directly in the object grpc will send (no intermediate buffer, no .tobytes())."""
    obj = _PyBytes_FromStringAndSize(None, n)
    return obj, _PyBytes_AsString(obj)


_tls = threading.local()


_CLASSIFY_NAME, _REGRESS_NAME = "tensorflow/serving/classify", "tensorflow/serving/regress"   # TF's signature_constants


def _method_kind(method) -> int:
    """RESP_CLASSIFY / RESP_REGRESS of a MultiInference task's method name; ValueError for any other."""
    if method == _CLASSIFY_NAME:
        return N.RESP_CLASSIFY
    if method == _REGRESS_NAME:
        return N.RESP_REGRESS
    raise ValueError(f"method {method!r} is neither {_CLASSIFY_NAME!r} nor {_REGRESS_NAME!r}")


def get_codec(device: int = 0) -> Codec:
    """Per-thread codec on `device` (contexts are not re-entrant)."""
    table = getattr(_tls, "codecs", None)
    if table is None:
        table = _tls.codecs = {}
    c = table.get(device)
    if c is None:
        c = table[device] = Codec(device)
    return c
