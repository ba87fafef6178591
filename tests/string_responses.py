"""PredictResponses with DT_STRING outputs, and the definition of their concatenated byte column, for the string decode tests
(tests/test_concat_strings_cpu.py, tests/test_concat_strings_gpu.py); strings_body is also the string_val payload the padded encode
tests expect (tests/test_padded_strings_cpu.py).

The definition: for a requested key, record r contributes S_r = list(PredictResponse.FromString(w_r).outputs[key].string_val)
(raw bytes) of shape dims_r (one -1 inferred); the column has shape (sum_r dims_r[0], *dims[1:]), int64 offsets[m + 1] from 0 and
the m strings of S_0 + S_1 + ... in its data.  A record without the key raises KeyError; another dtype, rank or trailing dims, rank
0 or len(S_r) != prod(dims_r) ValueError; malformed wire DecodeError.
"""
from typing import List, Sequence, Tuple

import numpy as np

import golden_util as G

DT_FLOAT, DT_STRING, DT_INT64 = 1, 7, 9


def strings_body(strs: Sequence[bytes]) -> bytes:
    """The string_val values on the wire: 42 vi(len) bytes per string."""
    return b"".join(G.ld(0x42, s) for s in strs)


def string_tensor(strs: Sequence[bytes], dims, *, dtype_last=False, unknown=False) -> bytes:
    """A DT_STRING TensorProto.  dtype_last: string_val and the shape before the dtype; unknown: unknown fields between the
    elements (a varint, a fixed64 and a length-delimited one)."""
    body = strings_body(strs)
    if unknown:
        junk = b"\xB8\x06\x07" + b"\xC1\x06" + b"\x01" * 8 + b"\xAA\x06\x03abc"
        body = b"".join(junk + G.ld(0x42, s) for s in strs) + junk
    shape = G.ld(0x12, G.shape(*dims))
    if dtype_last:
        return body + shape + b"\x08" + G.vi(DT_STRING)
    return b"\x08" + G.vi(DT_STRING) + shape + body


def float_tensor(x: np.ndarray) -> bytes:
    return G.tproto(DT_FLOAT, list(x.shape), G.ld(0x2A, np.ascontiguousarray(x, np.float32).tobytes()))


def int64_tensor(x: np.ndarray) -> bytes:
    from decode_mutants import packed_varints

    return G.tproto(DT_INT64, list(x.shape), G.ld(0x52, packed_varints(np.ascontiguousarray(x, np.int64).ravel().view(np.uint64))))


def response(*entries: Tuple[str, bytes], spec=True) -> bytes:
    """A PredictResponse of (key, TensorProto bytes) entries, in order, and a model_spec."""
    return b"".join(G.entry(k, tp) for k, tp in entries) + (G.mspec() if spec else b"")


def random_strings(rng: np.random.Generator, n: int, lo: int, hi: int) -> List[bytes]:
    """n strings of lo..hi bytes, every byte value (NUL and 0x80-0xFF included) equally likely."""
    lens = rng.integers(lo, hi + 1, n)
    return [rng.integers(0, 256, int(k), dtype=np.uint8).tobytes() for k in lens]


def reference(wires: Sequence[bytes], key: str):
    """(data uint8, offsets int64, shape) of the key's column, or the exception the definition raises."""
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
    if len({len(p[1]) for p in parts}) > 1 or len({p[1][1:] for p in parts}) > 1:
        raise ValueError("rank / trailing dims differ")
    strs = [s for p in parts for s in p[0]]
    offsets = np.zeros(len(strs) + 1, np.int64)
    np.cumsum([len(s) for s in strs], out=offsets[1:])
    data = np.frombuffer(b"".join(strs), np.uint8)
    return data, offsets, (sum(p[1][0] for p in parts),) + tuple(parts[0][1][1:])


def outcome(fn):
    """fn()'s result, or the type of the exception it raised."""
    try:
        return fn()
    except Exception as e:  # noqa: BLE001 - the type is what the tests compare
        return type(e)
