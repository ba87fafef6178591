"""The definition of the padded encode with string columns, built with the protobuf runtime: request r's string input is a DT_STRING
TensorProto of its box's raw bytes in C order, its numeric inputs what the protobuf runtime makes of the sliced arrays.  Shared by
the CPU and GPU tests of string inputs and by tools/padded_encode_probe.py."""
import numpy as np

from tensorflow.core.framework import tensor_pb2, tensor_shape_pb2, types_pb2
from tensorflow_serving.apis import predict_pb2

_NUMERIC = {np.dtype(np.float32): (types_pb2.DT_FLOAT, "float_val"), np.dtype(np.float64): (types_pb2.DT_DOUBLE, "double_val"),
            np.dtype(np.int32): (types_pb2.DT_INT32, "int_val"), np.dtype(np.int64): (types_pb2.DT_INT64, "int64_val"),
            np.dtype(np.bool_): (types_pb2.DT_BOOL, "bool_val")}


def _shape(dims):
    return tensor_shape_pb2.TensorShapeProto(dim=[tensor_shape_pb2.TensorShapeProto.Dim(size=int(d)) for d in dims])


def string_proto(strings, dims) -> tensor_pb2.TensorProto:
    return tensor_pb2.TensorProto(dtype=types_pb2.DT_STRING, tensor_shape=_shape(dims), string_val=list(strings))


def numeric_proto(a: np.ndarray) -> tensor_pb2.TensorProto:
    dt, field = _NUMERIC[a.dtype]
    p = tensor_pb2.TensorProto(dtype=dt, tensor_shape=_shape(a.shape))
    getattr(p, field).extend(a.ravel().tolist())
    return p


def request_wire(name, version, protos: dict, order="deterministic", grpc=False) -> bytes:
    """PredictRequest bytes: map entries sorted (deterministic) or in the dict's order ("given")."""
    spec = predict_pb2.PredictRequest()
    spec.model_spec.name = name
    if version is not None:
        spec.model_spec.version.value = version
    if order == "given":
        w = spec.SerializeToString() + b"".join(predict_pb2.PredictRequest(inputs={k: p}).SerializeToString() for k, p in protos.items())
    else:
        for k, p in protos.items():
            spec.inputs[k].CopyFrom(p)
        w = spec.SerializeToString(deterministic=True)
    return (b"\0" + len(w).to_bytes(4, "big") + w) if grpc else w


def random_column(rng, dims, max_len=40, alphabet=256):
    """(data uint8, offsets int64[m + 1], strings) of a column of shape dims with NUL and high bytes."""
    m = int(np.prod(dims, dtype=np.int64))
    lens = rng.integers(0, max_len + 1, m)
    data = rng.integers(0, alphabet, int(lens.sum())).astype(np.uint8)
    off = np.zeros(m + 1, np.int64)
    np.cumsum(lens, out=off[1:])
    return data, off, [data[off[j]: off[j + 1]].tobytes() for j in range(m)]


def box_strings(strings, dims, r0, row):
    """Strings of the box [r0 : r0 + row[0], :row[1], ...] of a column of shape dims, C order, and the box's dims."""
    bd = [int(row[0])] + ([int(x) for x in row[1:]] if len(row) > 1 else [int(d) for d in dims[1:]])
    idx = np.arange(len(strings)).reshape(dims)[(slice(r0, r0 + bd[0]),) + tuple(slice(0, x) for x in bd[1:])]
    return [strings[i] for i in idx.ravel().tolist()], bd


def reference_requests(name, version, padded: dict, shapes: dict, broadcast: dict, order="deterministic", grpc=False):
    """Every request's wire.  padded / broadcast values: numpy arrays, or (strings, dims) of a string column; shapes: int[n, m] or
    int[n] per padded key."""
    S = {k: np.asarray(s, np.int64).reshape(len(s), -1) for k, s in shapes.items()}
    n = len(next(iter(S.values())))
    r0 = {k: np.concatenate([[0], np.cumsum(s[:, 0])]) for k, s in S.items()}
    out = []
    for r in range(n):
        protos = {}
        for k, v in padded.items():
            row = S[k][r]
            if isinstance(v, tuple):
                strs, bd = box_strings(v[0], v[1], int(r0[k][r]), row)
                protos[k] = string_proto(strs, bd)
            else:
                box = (slice(int(r0[k][r]), int(r0[k][r]) + int(row[0])),) + tuple(slice(0, int(x)) for x in row[1:])
                protos[k] = numeric_proto(np.ascontiguousarray(v[box]))
        for k, v in broadcast.items():
            protos[k] = string_proto(v[0], v[1]) if isinstance(v, tuple) else numeric_proto(np.asarray(v))
        out.append(request_wire(name, version, protos, order, grpc))
    return out
