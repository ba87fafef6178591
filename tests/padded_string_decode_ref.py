"""The definition of a padded DT_STRING column of a batch of PredictResponses (Codec.decode_predict_responses_padded with
string_columns=True, b200tfs_decode_padded_strings), for tests/test_padded_string_decode_cpu.py and
tests/test_padded_string_decode_gpu.py.

For a requested key, response r contributes S_r = list(PredictResponse.FromString(w_r).outputs[key].string_val) (raw bytes) of
shape dims_r (one -1 inferred).  With tail = pad_to if given, else the elementwise maximum of dims_r[1:], the column has shape
(sum_r dims_r[0], *tail) in C order: response r's rows follow those of the responses before it, a position inside dims_r holds
its string and every other position of its rows holds `pad`.  offsets is int64[m + 1] from 0 and data the m strings one after the
other.  A response without the key raises KeyError; rank 0, another rank or dtype, a part larger than pad_to or a string count
that does not fill the shape ValueError; malformed wire DecodeError.
"""
from typing import Optional, Sequence

import numpy as np

DT_STRING = 7


def reference(wires: Sequence[bytes], key: str, pad: bytes = b"", pad_to: Optional[Sequence[int]] = None):
    """(data uint8, offsets int64, shape, shapes int64[n, rank]) of the key's padded column, or the exception the definition raises."""
    from tensorflow_serving.apis import predict_pb2

    parsed = [predict_pb2.PredictResponse.FromString(bytes(w)) for w in wires]
    parts = []
    for r in parsed:
        if key not in r.outputs:
            raise KeyError(key)
        t = r.outputs[key]
        if t.dtype != DT_STRING:
            from min_tfs_client import _native as N

            if not N.load().b200tfs_dtype_field(t.dtype):
                raise KeyError(t.dtype)       # what the per-response decode raises for a dtype it has no field for
            raise ValueError(f"dtype {t.dtype}")
        dims = [int(d.size) for d in t.tensor_shape.dim]
        if not dims:
            raise ValueError("rank 0")
        S = list(t.string_val)
        parts.append((S, np.empty(len(S), np.uint8).reshape(dims).shape))    # ValueError when the count does not fit
    rank = len(parts[0][1])
    if any(len(p[1]) != rank for p in parts):
        raise ValueError("ranks differ")
    tail = tuple(int(x) for x in pad_to) if pad_to is not None else tuple(max(p[1][d] for p in parts) for d in range(1, rank))
    if len(tail) != rank - 1 or any(p[1][d] > tail[d - 1] for p in parts for d in range(1, rank)):
        raise ValueError("does not fit pad_to")
    strs = []
    for S, shape in parts:
        own = np.empty(len(S), object)
        own[:] = S
        own = own.reshape(shape)
        for row in range(shape[0]):
            for idx in np.ndindex(*tail):
                inside = all(i < d for i, d in zip(idx, shape[1:]))
                strs.append(own[(row,) + idx] if inside else pad)
    offsets = np.zeros(len(strs) + 1, np.int64)
    np.cumsum([len(s) for s in strs], out=offsets[1:])
    data = np.frombuffer(b"".join(strs), np.uint8)
    shapes = np.array([p[1] for p in parts], np.int64).reshape(len(parts), rank)
    return data, offsets, (sum(p[1][0] for p in parts),) + tail, shapes


def strings_of(data, offsets):
    """The column's strings, in position order."""
    data, offsets = np.asarray(data), np.asarray(offsets)
    return [data[int(a): int(b)].tobytes() for a, b in zip(offsets[:-1], offsets[1:])]
