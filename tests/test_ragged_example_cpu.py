"""Ragged (variable-length) tf.Example columns without a GPU: the b200tfs_ragged mirror, the arena bound against the reference
bytes, the refusals of the ragged entry points (checked before the context is looked at), and RaggedColumn's own checks."""
import ctypes as C

import numpy as np
import pytest

from min_tfs_client import _native as N
from min_tfs_client.codec import RaggedColumn, _example_columns
from min_tfs_client.requests import examples_from_input_dict
from ragged_ref import ragged_ref

KEYS = ["a", "ab", "abc", "", "été", "中"]
ALL = [np.float16, np.float32, np.float64, np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint16, np.uint32, np.uint64, np.bool_]


def _values(rng, dt, shape):
    if np.dtype(dt).kind == "f":
        return rng.standard_normal(shape).astype(dt)
    if dt is np.bool_:
        return rng.integers(0, 2, shape).astype(np.bool_)
    info = np.iinfo(dt)
    return rng.integers(info.min, info.max, shape, dtype=dt, endpoint=True)


def _struct(d, grpc_frame=False):
    n, preps = _example_columns(d)
    feats = (N.Feature * max(len(preps), 1))(*[p[0] for p in preps])
    rg = (N.Ragged * max(len(preps), 1))(*[p[3] or N.Ragged() for p in preps])
    req = N.ExampleRequest(model_name=b"m", model_name_len=1, has_version=1, order=N.ORDER_UPB, version=2, n_examples=n,
                           n_features=len(preps), flags=N.RF_GRPC_FRAME if grpc_frame else 0, features=feats)
    return req, rg, (preps, feats)


def _ragged_host_rc(req, rg):
    """the ragged _host entry point with no context: its argument checks, or E_ARG for the missing context"""
    off, ln = (C.c_uint64 * 1)(), (C.c_uint64 * 1)()
    buf = C.create_string_buffer(16)
    rc = N.load().b200tfs_encode_example_requests_ragged_host(None, 1, C.byref(req), rg, buf, 16, off, ln)
    return rc, N.last_error()


def test_ragged_mirror_size():
    assert C.sizeof(N.Ragged) == 32
    assert [f[0] for f in N.Ragged._fields_] == ["lengths", "max_len", "unit", "flags", "pad_"]
    assert N.Ragged.max_len.offset == 8 and N.Ragged.unit.offset == 16 and N.Ragged.flags.offset == 24


@pytest.mark.parametrize("seed", range(24))
def test_arena_bounds_ragged_requests(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.choice([1, 9, 200]))
    d = {}
    for k in rng.choice(KEYS, size=int(rng.integers(1, 5)), replace=False):
        dt = ALL[int(rng.integers(len(ALL)))]
        L = int(rng.choice([0, 1, 5, 40]))
        inner = [(), (3,), (0,), (2, 2)][int(rng.integers(4))]
        lengths = rng.integers(0, L + 1, n)
        lengths[: min(n, 2)] = [0, L][: min(n, 2)]
        d[str(k)] = RaggedColumn(_values(rng, dt, (n, L) + inner), lengths.astype(rng.choice([np.int8, np.int32, np.uint16, np.int64])))
    if seed % 3 == 0:
        d["dense"] = rng.standard_normal((n, 3)).astype(np.float32)
        d["zero_d"] = np.int64(-1)
    d["neg"] = RaggedColumn(np.full((n, 6), -1, np.int64), np.full(n, 6))     # ten bytes per element: the worst case
    req, rg, keep = _struct(d, grpc_frame=bool(seed % 2))
    arena = C.c_uint64()
    N.check(N.load().b200tfs_example_arena_size(1, C.byref(req), C.byref(arena)))
    assert arena.value >= len(ragged_ref("m", 2, d, grpc_frame=bool(seed % 2)))


def test_ragged_entry_refusals():
    x = np.zeros((4, 6), np.float32)
    req, rg, keep = _struct({"x": RaggedColumn(x, [0, 1, 3, 2])})
    rc, msg = _ragged_host_rc(req, rg)
    assert rc == N.E_ARG and "context" in msg                 # well-formed: only the context is missing
    rg[0].unit = 2                                            # 6 != 6 * 2
    assert _ragged_host_rc(req, rg)[0] == N.E_ARG
    rg[0].unit, rg[0].max_len = 2, 3                          # 3 * 2 == 6: well-formed again
    assert "context" in _ragged_host_rc(req, rg)[1]
    rg[0].unit, rg[0].max_len = -1, -6
    assert _ragged_host_rc(req, rg)[0] == N.E_ARG
    rg[0].unit, rg[0].max_len = 0, 6                          # unit 0 needs row_elems 0
    assert _ragged_host_rc(req, rg)[0] == N.E_ARG
    rg[0].unit, rg[0].max_len = 1, 6
    rg[0].flags = 0x40
    assert _ragged_host_rc(req, rg)[0] == N.E_ARG
    rg[0].flags = 0
    req.features[0].flags = N.F_BROADCAST                     # a broadcast column cannot be ragged
    rc, msg = _ragged_host_rc(req, rg)
    assert rc == N.E_ARG and "broadcast" in msg
    req.features[0].flags = 0
    bad = np.array([0, 7, 1, 1], np.int64)                    # host lengths past max_len: refused before any launch
    rg[0].lengths = bad.ctypes.data
    assert _ragged_host_rc(req, rg)[0] == N.E_SHAPE
    bad[1] = -1
    assert _ragged_host_rc(req, rg)[0] == N.E_SHAPE
    empty = N.Feature(data=None, src_dtype=1, flags=0, row_elems=0, key=b"e", key_len=1)
    req.features, req.n_examples = C.pointer(empty), 4
    zero = np.zeros(4, np.int64)
    rg0 = (N.Ragged * 1)(N.Ragged(lengths=zero.ctypes.data, max_len=5, unit=0, flags=0))    # unit 0: rows of no elements
    assert "context" in _ragged_host_rc(req, rg0)[1]


def test_ragged_column_checks():
    v = np.zeros((3, 4, 2), np.int32)
    for bad in ([0, 5, 1], [-1, 0, 0], [0, 1], [[0, 1, 2]], [0.0, 1.0, 2.0]):
        with pytest.raises(ValueError):
            RaggedColumn(v, np.array(bad))
    with pytest.raises(ValueError):
        RaggedColumn(np.zeros(3, np.int32), [0, 0, 0])        # rank < 2
    with pytest.raises(ValueError):
        RaggedColumn(np.int32(1), [])
    ok = RaggedColumn(v, np.array([0, 4, 2], np.uint8))
    assert ok.lengths.dtype == np.int64 and ok.ndim == 3
    with pytest.raises(ValueError, match="disagree"):
        examples_from_input_dict({"r": ok, "d": np.zeros(4)})
    with pytest.raises(ValueError, match="disagree"):
        _example_columns({"r": ok, "d": np.zeros(4)})


def test_examples_from_input_dict_takes_ragged_columns():
    vals = np.arange(24, dtype=np.int64).reshape(3, 4, 2)
    inp = examples_from_input_dict({"r": RaggedColumn(vals, [0, 4, 1]), "s": RaggedColumn(np.array([["a", "b"], ["c", "d"], ["e", "f"]]), [2, 0, 1]),
                                    "x": np.float32(1.5)})
    ex = inp.example_list.examples
    assert [list(e.features.feature["r"].int64_list.value) for e in ex] == [[], list(range(8, 16)), [16, 17]]
    assert [list(e.features.feature["s"].bytes_list.value) for e in ex] == [[b"a", b"b"], [], [b"e"]]
    assert all(e.features.feature["x"].float_list.value == [1.5] for e in ex)


def test_example_columns_builds_ragged_structs():
    vals = np.zeros((5, 7, 3, 2), np.float64)
    lengths = np.array([0, 7, 3, 1, 2], np.int16)
    n, preps = _example_columns({"r": RaggedColumn(vals, lengths), "d": np.zeros((5, 2), np.int8), "c": np.float32(1)})
    assert n == 5 and len(preps) == 3
    f, hold, key, g = preps[0]
    assert key == b"r" and f.row_elems == 42 and f.flags == 0 and f.src_dtype == 2
    assert g.max_len == 7 and g.unit == 6 and g.flags == 0
    assert np.ctypeslib.as_array((C.c_int64 * 5).from_address(g.lengths)).tolist() == lengths.tolist()
    assert preps[1][3] is None and preps[2][3] is None and preps[2][0].flags == N.F_BROADCAST
    assert _example_columns({"s": RaggedColumn(np.array([["x"]]), [1])}) is None         # strings: the host route
