"""String (bytes_list) tf.Example columns without a GPU: the b200tfs_bytes mirror, the refusals of the *_example_columns_* entry
points (checked before the context is looked at), BytesColumn.from_array against the host route's string conversion, the host
reference of a BytesColumn, and the arena bound against the protobuf size of random requests."""
import ctypes as C

import numpy as np
import pytest

from min_tfs_client import _native as N
from min_tfs_client.codec import BytesColumn, RaggedColumn, _example_columns
from min_tfs_client.requests import TensorServingClient, examples_from_input_dict
from min_tfs_client.tensors import coerce_to_bytes
from tensorflow_serving.apis.classification_pb2 import ClassificationRequest


def _ref(d, version=2, grpc_frame=False):
    wire = TensorServingClient._make_example_request(None, ClassificationRequest, "m", d, version).SerializeToString(deterministic=True)
    return (b"\x00" + len(wire).to_bytes(4, "big") + wire) if grpc_frame else wire


def _struct(d, grpc_frame=False):
    n, preps = _example_columns(d)
    feats = (N.Feature * max(len(preps), 1))(*[p[0] for p in preps])
    rg = (N.Ragged * max(len(preps), 1))(*[p[3] or N.Ragged() for p in preps])
    bs = (N.Bytes * max(len(preps), 1))(*[p.bytes_entry or N.Bytes() for p in preps])
    req = N.ExampleRequest(model_name=b"m", model_name_len=1, has_version=1, order=N.ORDER_UPB, version=2, n_examples=n,
                           n_features=len(preps), flags=N.RF_GRPC_FRAME if grpc_frame else 0, features=feats)
    return req, rg, bs, (preps, feats)


def _host_rc(req, rg, bs):
    """the columns _host entry point with no context: its argument checks, or E_ARG for the missing context"""
    off, ln = (C.c_uint64 * 1)(), (C.c_uint64 * 1)()
    buf = C.create_string_buffer(16)
    rc = N.load().b200tfs_encode_example_columns_host(None, 1, C.byref(req), rg, bs, None, buf, 16, off, ln)
    return rc, N.last_error()


def _async_rc(req, bs):
    buf = C.create_string_buffer(16)
    return N.load().b200tfs_encode_example_columns_async(None, 1, C.byref(req), None, bs, None, buf, 16)


def _size_rc(req, bs):
    out = C.c_uint64()
    return N.load().b200tfs_example_columns_arena_size(1, C.byref(req), bs, None, C.byref(out))


def _strings(rng, m, lo=0, hi=12):
    alphabet = np.frombuffer(bytes(range(256)), np.uint8)
    return [rng.choice(alphabet, int(rng.integers(lo, hi + 1))).tobytes() for _ in range(m)]


def _column(strs, shape=None, start=0):
    """a BytesColumn of these strings, its buffer `start` bytes in (offsets[0] == start)"""
    lens = np.array([len(s) for s in strs], np.int64)
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64) + start
    data = np.frombuffer(b"\xEE" * start + b"".join(strs) + b"\xEE" * 3, np.uint8)
    return BytesColumn(data, offsets, shape)


def test_bytes_mirror():
    assert C.sizeof(N.Bytes) == 24
    assert [f[0] for f in N.Bytes._fields_] == ["offsets", "data_len", "flags", "pad_"]
    assert N.Bytes.data_len.offset == 8 and N.Bytes.flags.offset == 16


def test_entry_refusals():
    rng = np.random.default_rng(1)
    col = _column(_strings(rng, 12), (4, 3))
    req, rg, bs, keep = _struct({"s": col, "x": np.zeros((4, 2), np.float32)})
    rc, msg = _host_rc(req, rg, bs)
    assert rc == N.E_ARG and "context" in msg                 # well-formed: only the context is missing
    assert _async_rc(req, bs) == N.E_ARG and "bad arguments" in N.last_error()
    assert _size_rc(req, bs) == N.OK
    saved = N.Bytes(bs[0].offsets, bs[0].data_len, bs[0].flags)
    for field, value in (("flags", 0x40), ("data_len", -1), ("offsets", saved.offsets + 4)):
        setattr(bs[0], field, value)
        assert _host_rc(req, rg, bs)[0] == N.E_ARG, field
        assert _async_rc(req, bs) == N.E_ARG and "feature 0" in N.last_error(), field
        assert _size_rc(req, bs) == N.E_ARG, field
        bs[0] = saved
    bs[1] = N.Bytes(offsets=saved.offsets, data_len=1, flags=0)        # an entry on the float column
    rc, msg = _host_rc(req, rg, bs)
    assert rc == N.E_ARG and "dtype" in msg
    assert _async_rc(req, bs) == N.E_ARG
    bs[1] = N.Bytes()
    bs[0] = N.Bytes()                                                   # a DT_STRING column without an entry
    assert _host_rc(req, rg, bs)[0] == N.E_DTYPE
    assert _async_rc(req, bs) == N.E_DTYPE
    assert _size_rc(req, bs) == N.E_DTYPE
    bs[0] = saved
    # the entry points without bytes entries still refuse a DT_STRING column as before
    out = C.c_uint64()
    assert N.load().b200tfs_example_arena_size(1, C.byref(req), C.byref(out)) == N.E_DTYPE
    assert _host_rc(req, rg, None)[0] == N.E_DTYPE


@pytest.mark.parametrize("case", ["decreasing", "negative", "past_data_len", "row_start_past_next", "ragged_end_past_next"])
def test_host_offsets_breaking_the_rule_are_refused(case):
    strs = [b"ab", b"", b"cde", b"f", b"gh", b"ij"]
    col = _column(strs, (3, 2))
    o = col.offsets
    lengths = None
    if case == "decreasing":
        o[3] = o[2] - 1
    elif case == "negative":
        o[0] = -1
    elif case == "past_data_len":
        o[6] = col.data_len + 1
    elif case == "row_start_past_next":
        o[2], o[3] = o[4] + 1, o[4] + 1
    else:                                                      # a ragged row's last string ends past the next row's start
        lengths = np.array([1, 2, 2])
        o[1] = o[2] + 1
    d = {"s": col if lengths is None else RaggedColumn(col, lengths)}
    req, rg, bs, keep = _struct(d)
    rc, msg = _host_rc(req, rg, bs)
    assert rc == N.E_SHAPE and "offsets" in msg, msg
    ok = {"s": _column(strs, (3, 2))}
    req, rg, bs, keep = _struct(ok)
    assert "context" in _host_rc(req, rg, bs)[1]


def test_ragged_padding_strings_are_not_read():
    """strings past a ragged row's length are padding: their offsets may hold anything up to the next row's start"""
    col = _column([b"ab", b"c", b"d", b"ef", b"g", b""], (2, 3))
    col.offsets[2] = 0                                          # the end of string 1 of row 0 (padding for length 1) goes backwards
    req, rg, bs, keep = _struct({"s": RaggedColumn(col, [1, 3])})
    assert "context" in _host_rc(req, rg, bs)[1]


def _coerced(a):
    return [coerce_to_bytes(s) for s in np.asarray(a).ravel().tolist()]


@pytest.mark.parametrize("a", [
    np.array([b"x\x00", b"a\x00b", b"", b"\x00", b"\xff\x80", b"plain"]),
    np.array([["été", ""], ["中文字", "a\x00b"], ["x\x00", "\U0001F600"]]),
    np.array("zero-d"),
    np.array(b"\x00\x01\x00"),
    np.array([], dtype="U4"),
    np.array([[b""] * 3] * 2),
    np.array(["ascii", "é" * 50, ""]).reshape(3, 1, 1),
], ids=lambda a: f"{a.dtype}{a.shape}")
def test_from_array_matches_coerce_to_bytes(a):
    col = BytesColumn.from_array(a)
    assert col.shape == a.shape and col.data.dtype == np.uint8 and col.offsets.dtype == np.int64
    got = [bytes(col.data[col.offsets[j]: col.offsets[j + 1]]) for j in range(col.offsets.size - 1)]
    assert got == _coerced(a)
    assert col.data_len == sum(len(s) for s in got)


def test_from_array_surrogate_raises_like_the_host_route():
    a = np.array(["ok", "bad\ud800"])
    with pytest.raises(UnicodeEncodeError) as host:
        examples_from_input_dict({"s": a})
    with pytest.raises(UnicodeEncodeError) as mine:
        BytesColumn.from_array(a)
    assert str(mine.value) == str(host.value)
    with pytest.raises(ValueError):
        BytesColumn.from_array(np.arange(3))


def test_column_checks():
    with pytest.raises(ValueError):
        BytesColumn(np.zeros(4, np.uint8), np.array([0, 1, 2]), (3,))     # 2 strings do not fill 3
    with pytest.raises(ValueError):
        BytesColumn(np.zeros(4, np.int8), np.array([0, 4]))               # data is not uint8
    with pytest.raises(ValueError):
        BytesColumn(np.zeros(4, np.uint8), np.array([0.0, 4.0]))          # offsets are not integers
    with pytest.raises(ValueError):
        BytesColumn(np.zeros(4, np.uint8), np.zeros(0, np.int64))         # no offsets at all
    c = BytesColumn(b"abcd", np.array([1, 3], np.int32), ())
    assert c.shape == () and c.offsets.dtype == np.int64 and c.strings(5) == [b"bc"]
    assert BytesColumn(b"", [0]).shape == (0,)


@pytest.mark.parametrize("seed", range(6))
def test_host_reference_equals_numpy_strings(seed):
    """examples_from_input_dict of a BytesColumn is the request of the same strings as a numpy str / bytes array"""
    rng = np.random.default_rng(seed)
    n = int(rng.choice([1, 7, 40]))
    words = np.array(["", "a", "été", "中文", "x\x00y", "longer word here"])
    u = rng.choice(words, (n, 3))
    s = np.array([b"", b"\x01\xff", b"a\x00b", b"zz"])[rng.integers(0, 4, n)]
    d_np = {"u": u, "s": s, "c": np.array("country"), "f": rng.standard_normal((n, 2)).astype(np.float32)}
    d_col = {"u": BytesColumn.from_array(u), "s": BytesColumn.from_array(s), "c": BytesColumn.from_array(np.array("country")),
             "f": d_np["f"]}
    assert _ref(d_col) == _ref(d_np)
    assert _example_columns(d_np) is None and _example_columns(d_col) is not None


def _rand_request(rng):
    n = int(rng.choice([0, 1, 9, 120]))
    d = {}
    for k in range(int(rng.integers(1, 4))):
        kind = int(rng.integers(4))
        inner = int(rng.choice([0, 1, 3]))
        hi = int(rng.choice([0, 5, 200, 300]))
        if kind == 0:
            d[f"b{k}"] = _column(_strings(rng, n * inner, 0, hi), (n, inner), start=int(rng.integers(0, 9)))
        elif kind == 1:
            d[f"z{k}"] = _column(_strings(rng, 1, 0, hi), ())
        elif kind == 2:
            L = int(rng.choice([1, 4]))
            lengths = rng.integers(0, L + 1, n)
            lengths[: min(n, 1)] = L
            d[f"r{k}"] = RaggedColumn(_column(_strings(rng, n * L * max(inner, 1), 0, hi), (n, L, max(inner, 1))), lengths)
        else:
            d[f"i{k}"] = np.full((n, inner), -1, np.int64)
    d["x"] = rng.standard_normal((n, 2)).astype(np.float32)
    return d


@pytest.mark.parametrize("seed", range(30))
def test_arena_bound_covers_the_request(seed):
    rng = np.random.default_rng(100 + seed)
    items = [_rand_request(rng) for _ in range(int(rng.integers(1, 4)))]
    frame = bool(seed % 2)
    structs = [_struct(d, grpc_frame=frame) for d in items]
    reqs = (N.ExampleRequest * len(items))(*[s[0] for s in structs])
    bs = (N.Bytes * sum(max(s[0].n_features, 0) for s in structs))(*[b for s in structs for b in list(s[2])[: s[0].n_features]])
    cap = C.c_uint64()
    N.check(N.load().b200tfs_example_columns_arena_size(len(items), reqs, bs, None, C.byref(cap)))
    need = 0
    for d in items:                                   # each slot starts 256-byte aligned, its examples behind a 16-aligned anchor
        need = ((need + 255) & ~255) + len(_ref(d, grpc_frame=frame)) + 16
    assert cap.value >= need
