"""A numpy writer of SequenceExample Predict requests built from the field numbers alone (no protobuf): what
requests.make_predict_sequence_examples_request + SerializeToString(deterministic=True) give.

    sequence   = 0A vi(C) {context map entries} 12 vi(G) {0A vi(e) 0A vi(klen) key 12 vi(FL) {0A vi(feat) Feature}*}*
    Feature    = 12 vi(list) [0A vi(P) f32...] | 1A vi(list) [0A vi(P) varints] | 0A vi(P) {0A vi(len) bytes}*

Each sequence's payloads are cut from the columns with numpy, so cases scale to tens of thousands of sequences."""
import numpy as np

from example_ref import _f32_bits, _i64, prefix, upb_order, varints, vi
from min_tfs_client.codec import BytesColumn, RaggedColumn


def _field(tag: int, body: bytes) -> bytes:
    return bytes([tag]) + vi(len(body)) + body


def _feature(kind: str, vals) -> bytes:
    """the Feature message of one row (float / int values, or a list of strings)"""
    if kind == "bytes":
        return _field(0x0A, b"".join(_field(0x0A, s) for s in vals))
    if kind == "float":
        payload = _f32_bits(vals).tobytes()
        return _field(0x12, _field(0x0A, payload) if payload else b"")
    payload = varints(_i64(vals))[1].tobytes() if len(vals) else b""
    return _field(0x1A, _field(0x0A, payload) if payload else b"")


class _Value:
    """one value of a context or feature-list dict: its kind, and the flat elements (or strings) of any run of its rows"""

    def __init__(self, key, v):
        self.key = key.encode("utf-8") if isinstance(key, str) else bytes(key)
        self.lengths = np.asarray(v.lengths).astype(np.int64) if isinstance(v, RaggedColumn) else None
        inner = v.values if isinstance(v, RaggedColumn) else v
        if isinstance(inner, BytesColumn):
            self.kind, self.shape = "bytes", tuple(inner.shape)
            self.data, self.off = np.asarray(inner.data).tobytes(), np.asarray(inner.offsets).astype(np.int64)
        else:
            a = np.asarray(inner)
            self.kind, self.shape = ("float" if a.dtype.kind == "f" else "int"), a.shape
            self.flat = a.reshape(-1)
        self.row = int(np.prod(self.shape[1:], dtype=np.int64)) if self.shape else 1
        self.unit = int(np.prod(self.shape[2:], dtype=np.int64)) if len(self.shape) >= 2 else 1

    def elems(self, start, count):
        if self.kind == "bytes":
            o = self.off[start: start + count + 1].tolist()
            return [self.data[o[j]: o[j + 1]] for j in range(count)]
        return self.flat[start: start + count]

    def context(self, i) -> bytes:
        """sequence i's context Feature (a 0-d value: its one element; ragged: the first lengths[i] * unit)"""
        if not self.shape:
            return _feature(self.kind, self.elems(0, 1))
        count = self.row if self.lengths is None else int(self.lengths[i]) * self.unit
        return _feature(self.kind, self.elems(i * self.row, count))

    def steps(self, i) -> bytes:
        """sequence i's FeatureList body: one 0A-tagged Feature per step"""
        T = self.shape[1] if self.lengths is None else int(self.lengths[i])
        return b"".join(_field(0x0A, _feature(self.kind, self.elems(i * self.row + t * self.unit, self.unit))) for t in range(T))


def n_sequences(context, feature_lists) -> int:
    rows = {tuple(_Value(k, v).shape)[0] for k, v in context.items() if len(_Value(k, v).shape)}
    rows |= {_Value(k, v).shape[0] for k, v in feature_lists.items()}
    assert len(rows) <= 1
    return rows.pop() if rows else (1 if context or feature_lists else 0)


def _ordered(d, order):
    vals = [_Value(k, v) for k, v in d.items()]
    return vals if order == "given" else [vals[i] for i in upb_order([v.key for v in vals])]


def sequences(context, feature_lists, order="deterministic"):
    """every sequence's serialized bytes"""
    n = n_sequences(context, feature_lists)
    cv, lv = _ordered(context, order), _ordered(feature_lists, order)
    out = []
    for i in range(n):
        C = b"".join(_field(0x0A, _field(0x0A, v.key) + _field(0x12, v.context(i))) for v in cv)
        G = b"".join(_field(0x0A, _field(0x0A, v.key) + _field(0x12, v.steps(i))) for v in lv)
        out.append(_field(0x0A, C) + _field(0x12, G))
    return out


def request_bytes(name, version, context, feature_lists, key, grpc=False, order="deterministic") -> bytes:
    """the PredictRequest whose input `key` is the DT_STRING [n] tensor of the sequences"""
    body = b"".join(_field(0x42, s) for s in sequences(context, feature_lists, order))
    return prefix(name, version, n_sequences(context, feature_lists), len(body), key, grpc) + body
