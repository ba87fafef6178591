"""ctypes front-end of the C oracle (``oracle/wire_oracle.c``).  TEST INFRASTRUCTURE ONLY.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl reference``
legs may import this module; the product (``min-tfs-client_b200/``) never does - it has no CPU path.
Parity status of the oracle: PINNED against the vectors the unmodified reference produced
(``tests/golden/*.json``; replayed by ``tests/test_oracle.py``).

numpy arrays in, ``bytes`` out (encode) and back (decode), same conventions as the reference:
C-order ravel, typed repeated fields, ``deterministic=True`` map order ("upb") for several inputs.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "liboracle.so")

OK, E_DTYPE, E_SHAPE, E_PARSE, E_RANGE, E_KEY, E_RANK0 = 0, -1, -2, -4, -9, -10, -20
F_CONTENT, F_KEEP_SNAN = 1, 2
MAX_RANK, MAX_OUT = 64, 64

_DT = {"float32": 1, "float64": 2, "int32": 3, "uint8": 4, "int16": 5, "int8": 6, "complex64": 8, "int64": 9, "bool": 10,
       "bfloat16": 14, "uint16": 17, "complex128": 18, "float16": 19, "uint32": 22, "uint64": 23}
_NP = {v: k for k, v in _DT.items()}
DT_STRING = 7


class _Tensor(C.Structure):
    _fields_ = [("data", C.c_void_p), ("src_dtype", C.c_int32), ("wire_dtype", C.c_int32), ("rank", C.c_int32), ("flags", C.c_int32),
                ("dims", C.POINTER(C.c_int64)), ("key", C.c_char_p), ("key_len", C.c_int64)]


class _Desc(C.Structure):
    _fields_ = [("key_off", C.c_int64), ("key_len", C.c_int64), ("dtype", C.c_int32), ("rank", C.c_int32), ("status", C.c_int32),
                ("pad", C.c_int32), ("dims", C.c_int64 * MAX_RANK), ("n_elems", C.c_int64), ("msg_off", C.c_int64), ("msg_len", C.c_int64)]


class _Spec(C.Structure):
    _fields_ = [("name_off", C.c_int64), ("name_len", C.c_int64), ("sig_off", C.c_int64), ("sig_len", C.c_int64),
                ("label_off", C.c_int64), ("label_len", C.c_int64), ("version", C.c_int64), ("has_version", C.c_int32), ("pad", C.c_int32)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(os.path.join(_HERE, "wire_oracle.c")):
            subprocess.run(["make", "-s", "-C", _HERE], check=True)
        L = C.CDLL(_SO)
        L.orc_tensor_proto.restype = C.c_int64
        L.orc_tensor_proto.argtypes = [C.POINTER(_Tensor), C.c_void_p]
        L.orc_predict_request.restype = C.c_int64
        L.orc_predict_request.argtypes = [C.c_char_p, C.c_int64, C.c_int, C.c_int64, C.c_int, C.POINTER(_Tensor), C.c_void_p]
        L.orc_predict_response.restype = C.c_int64
        L.orc_predict_response.argtypes = [C.c_char_p, C.c_int64, C.c_int64, C.c_char_p, C.c_int64, C.c_int, C.POINTER(_Tensor), C.c_void_p]
        L.orc_order_upb.restype = None
        L.orc_order_upb.argtypes = [C.c_int, C.POINTER(_Tensor), C.POINTER(C.c_int32)]
        L.orc_parse_response.restype = C.c_void_p
        L.orc_parse_response.argtypes = [C.c_void_p, C.c_int64, C.POINTER(_Desc), C.POINTER(C.c_int32), C.POINTER(_Spec)]
        L.orc_parse_tensor.restype = C.c_void_p
        L.orc_parse_tensor.argtypes = [C.c_void_p, C.c_int64, C.POINTER(_Desc)]
        L.orc_write_output.restype = C.c_int32
        L.orc_write_output.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        L.orc_free.restype = None
        L.orc_free.argtypes = [C.c_void_p]
        L.orc_content_len.restype = C.c_int64
        L.orc_content_len.argtypes = [C.c_void_p, C.c_int]
        L.orc_value_count.restype = C.c_int64
        L.orc_value_count.argtypes = [C.c_void_p, C.c_int]
        L.orc_content_off.restype = C.c_int64
        L.orc_content_off.argtypes = [C.c_void_p, C.c_int]
        for fn in (L.orc_narrow_f32, L.orc_widen_16):
            fn.restype = None
            fn.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int]
        L.orc_int_to_half.restype = None
        L.orc_int_to_half.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
        _lib = L
    return _lib


def _dt_of(arr: np.ndarray) -> int:
    name = arr.dtype.name
    if name not in _DT:
        raise ValueError(f"Dtype {name} is not valid")
    return _DT[name]


def _string_proto(arr: np.ndarray) -> bytes:
    """DT_STRING TensorProto by hand (small cases only): unpacked string_val elements."""
    def uv(x):
        out = bytearray()
        while True:
            b = x & 0x7F
            x >>= 7
            out.append(b | (0x80 if x else 0))
            if not x:
                return bytes(out)
    shape = b"".join(b"\x12" + (uv(1 + len(uv(d))) + b"\x08" + uv(d) if d else b"\x00") for d in arr.shape)
    body = b"\x08\x07\x12" + uv(len(shape)) + shape
    for s in arr.ravel().tolist():
        b = s.encode("utf-8") if isinstance(s, str) else s
        body += b"\x42" + uv(len(b)) + b
    return body


class _Prep:
    def __init__(self, arr, key=b"", wire_dtype=None, tensor_content=False, keep_snan=False):
        arr = np.asarray(arr)
        if not arr.dtype.isnative:
            arr = arr.astype(arr.dtype.newbyteorder("="))
        self.arr = np.ascontiguousarray(arr)
        self.dims = (C.c_int64 * max(arr.ndim, 1))(*arr.shape)
        src = _dt_of(self.arr)
        wire = src if wire_dtype is None else (wire_dtype if isinstance(wire_dtype, int) else _DT[np.dtype(wire_dtype).name])
        self.key = key
        self.t = _Tensor(self.arr.ctypes.data if self.arr.size else None, src, wire, arr.ndim,
                         (F_CONTENT if tensor_content else 0) | (F_KEEP_SNAN if keep_snan else 0), self.dims, key, len(key))


def _emit(fn, *args):
    n = fn(*args, None)
    if n < 0:
        raise ValueError(f"oracle error {n}")
    buf = C.create_string_buffer(int(n) or 1)
    m = fn(*args, buf)
    assert m == n
    return buf.raw[: int(n)]


def encode_tensor_proto(arr, **kw) -> bytes:
    arr = np.asarray(arr)
    if arr.dtype.kind == "U":
        return _string_proto(arr)
    p = _Prep(arr, **kw)
    return _emit(lib().orc_tensor_proto, C.byref(p.t))


def encode_predict_request(model_name, model_version, inputs, order="upb", **kw) -> bytes:
    """inputs: list of (key, ndarray).  order 'upb' = SerializeToString(deterministic=True) order."""
    name = model_name.encode("utf-8") if isinstance(model_name, str) else model_name
    preps = []
    for k, v in inputs:
        if np.asarray(v).dtype.kind == "U":
            raise ValueError("string inputs: use the reference port (oracle.ref_port) for those cases")
        preps.append(_Prep(v, key=k.encode("utf-8") if isinstance(k, str) else k, **kw))
    n = len(preps)
    ts = (_Tensor * max(n, 1))(*[p.t for p in preps])
    if order == "upb" and n > 1:
        perm = (C.c_int32 * n)()
        lib().orc_order_upb(n, ts, perm)
        ts = (_Tensor * n)(*[preps[i].t for i in perm])
    return _emit(lib().orc_predict_request, name, len(name), int(model_version is not None), int(model_version or 0), n, ts)


def build_predict_response(outputs, model_name="default", version=1, signature="serving_default", **kw) -> bytes:
    """Canonical tensorflow_model_server layout: outputs entries, then model_spec."""
    preps = [_Prep(v, key=k.encode("utf-8"), **kw) for k, v in outputs]
    ts = (_Tensor * max(len(preps), 1))(*[p.t for p in preps])
    name, sig = model_name.encode(), signature.encode()
    return _emit(lib().orc_predict_response, name, len(name), int(version), sig, len(sig), len(preps), ts)


_EXC = {E_SHAPE: ValueError, E_KEY: KeyError, E_RANK0: TypeError, E_RANGE: OverflowError, E_DTYPE: ValueError}
_RANGE_CHECKED = (4, 5, 6, 17)     # DT_UINT8, DT_INT16, DT_INT8, DT_UINT16: int_val values narrowed by np.array(values, dtype)


class ParseError(Exception):
    """What DecodeError is for the reference's FromString."""


def _materialise(handle, i, d: _Desc, wire: bytes, half_mode: int, tolerant: bool):
    if d.dtype == DT_STRING and d.status in (OK, E_RANK0):
        raise NotImplementedError("string outputs: use the reference port")
    status = d.status
    if tolerant and status == E_RANK0:
        status = OK
    if tolerant and status == E_SHAPE and d.dtype in _NP:  # tensor_content carries the values (TF convention)
        shape = tuple(d.dims[k] for k in range(d.rank))
        nb = int(np.prod(shape, dtype=np.int64)) * np.dtype(_np_dtype(d.dtype)).itemsize
        if lib().orc_content_len(handle, i) == nb and nb:
            off = lib().orc_content_off(handle, i)
            return np.frombuffer(wire[off: off + nb], dtype=_np_dtype(d.dtype)).reshape(shape).copy()
    if tolerant and status == E_SHAPE and d.dtype in _NP and lib().orc_content_len(handle, i):
        # MakeNdarray takes tensor_content whenever it is there (tensor_util.py:565-642 in the reference's vendored tree): bytes of
        # the wrong length do not reshape, and the typed values are never looked at (ref_port.make_ndarray_tf)
        raise ValueError("tensor_content does not match the shape")
    if tolerant and status == E_SHAPE and d.dtype in _NP:
        # TensorFlow's MakeNdarray (tensor_util.py:631-640 in the reference's vendored tree): no values -> zeros, fewer values
        # than the shape holds -> the last one repeats ("edge" padding); more values stays an error
        shape = tuple(d.dims[k] for k in range(d.rank))
        want = int(np.prod(shape, dtype=np.int64)) if all(s >= 0 for s in shape) else -1
        have = int(lib().orc_value_count(handle, i))
        if 0 <= have < want:
            flat = np.zeros(want, dtype=_np_dtype(d.dtype))
            if have:
                rc = lib().orc_write_output(handle, i, half_mode, flat.ctypes.data)
                if rc != OK:
                    raise _EXC.get(rc, ValueError)(f"oracle status {rc}")
                flat[have:] = flat[have - 1]
            return flat.reshape(shape)
    if status == E_SHAPE and d.dtype in _RANGE_CHECKED:
        # np.array(values, dtype) refuses an out-of-range value before reshape() refuses the element count
        have = int(lib().orc_value_count(handle, i))
        if have > 0:
            scratch = np.empty(have, dtype=_np_dtype(d.dtype))
            if lib().orc_write_output(handle, i, half_mode, scratch.ctypes.data) == E_RANGE:
                raise OverflowError(f"oracle status {E_RANGE}")
    if status != OK:
        raise _EXC.get(status, ValueError)(f"oracle status {status}")
    shape = tuple(d.dims[k] for k in range(d.rank))
    out = np.empty(shape, dtype=_np_dtype(d.dtype))
    rc = lib().orc_write_output(handle, i, half_mode, out.ctypes.data if out.size else None)
    if rc != OK:
        raise _EXC.get(rc, ValueError)(f"oracle status {rc}")
    return out


def _is_bf16(np_dtype) -> bool:
    name = np.dtype(np_dtype).name
    if name not in ("float16", "bfloat16"):
        raise ValueError(f"not a 16-bit float dtype: {name}")
    return name == "bfloat16"


def narrow_f32(x, np_dtype) -> np.ndarray:
    """float32 -> float16 / bfloat16 the way ``tensor_proto_to_ndarray(...).astype(np_dtype)`` narrows a decoded
    float32: NaNs quieted first (the reference's double trip), then round to nearest even, computed with integers."""
    bits = np.ascontiguousarray(np.asarray(x).view(np.uint32))
    out = np.empty(bits.shape, dtype=np.uint16)
    lib().orc_narrow_f32(bits.ctypes.data, out.ctypes.data, bits.size, int(_is_bf16(np_dtype)))
    return out.view(_np_dtype(_DT["bfloat16"]) if _is_bf16(np_dtype) else np.float16)


def widen_16(x) -> np.ndarray:
    """float16 / bfloat16 -> the float32 the reference puts on the wire for ``wire_dtype=DT_FLOAT`` (exact; NaNs quiet)."""
    x = np.ascontiguousarray(x)
    out = np.empty(x.shape, dtype=np.uint32)
    lib().orc_widen_16(x.view(np.uint16).ctypes.data, out.ctypes.data, x.size, int(_is_bf16(x.dtype)))
    return out.view(np.float32)


def int_to_half(v) -> np.ndarray:
    """int32 ``half_val`` values -> float16 values, round to nearest even (the reference's DT_HALF quirk)."""
    v = np.ascontiguousarray(v, dtype=np.int32)
    out = np.empty(v.shape, dtype=np.uint16)
    lib().orc_int_to_half(v.ctypes.data, out.ctypes.data, v.size)
    return out.view(np.float16)


def _np_dtype(enum):
    name = _NP[enum]
    if name == "bfloat16":
        import ml_dtypes

        return ml_dtypes.bfloat16
    return np.dtype(name)


def decode_predict_response(wire: bytes, *, strict=True, with_spec=False):
    """dict key -> ndarray as FromString + tensor_proto_to_ndarray give (strict), or with TF's
    conventions for what the reference rejects (strict=False)."""
    descs = (_Desc * MAX_OUT)()
    n = C.c_int32(0)
    spec = _Spec()
    buf = C.create_string_buffer(wire, len(wire))
    h = lib().orc_parse_response(buf, len(wire), descs, C.byref(n), C.byref(spec))
    if not h:
        raise ParseError("malformed PredictResponse")
    try:
        out = {}
        for i in range(n.value):
            d = descs[i]
            key = wire[d.key_off: d.key_off + d.key_len].decode("utf-8")
            if strict and d.dtype in (8, 18) and d.status == OK and d.n_elems:
                raise ValueError("reference reads complex values as separate floats")
            if strict and d.dtype == 14:
                raise KeyError(14)
            out[key] = _materialise(h, i, d, wire, 1 if strict else 0, not strict)
        if with_spec:
            s = {"name": wire[spec.name_off: spec.name_off + spec.name_len].decode(), "version": spec.version,
                 "has_version": bool(spec.has_version), "version_label": wire[spec.label_off: spec.label_off + spec.label_len].decode(),
                 "signature_name": wire[spec.sig_off: spec.sig_off + spec.sig_len].decode()}
            return out, s
        return out
    finally:
        lib().orc_free(h)


def decode_tensor_proto(wire: bytes, *, strict=True):
    d = _Desc()
    buf = C.create_string_buffer(wire, len(wire))
    h = lib().orc_parse_tensor(buf, len(wire), C.byref(d))
    if not h:
        raise ParseError("malformed TensorProto")
    try:
        if strict and d.dtype == 14:
            raise KeyError(14)
        return _materialise(h, 0, d, wire, 1 if strict else 0, not strict)
    finally:
        lib().orc_free(h)
