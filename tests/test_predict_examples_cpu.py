"""PredictRequests carrying serialized tf.Examples, without a GPU: the b200tfs_example_target mirror, the exact size against the
protobuf runtime's ByteSize(), the arena bound against the reference bytes, the refusals of the target entry points (checked
before the context is looked at) and the Python host route for a request with a str column."""
import ctypes as C

import numpy as np
import pytest

from min_tfs_client import _native as N
from min_tfs_client.codec import RaggedColumn, _example_columns, _host_example_request
from predict_examples_ref import predict_examples_ref, predict_examples_request

KEYS = ["examples", "", "a", "ab", "inputs", "input", "été", "中文", "k" * 200]
ALL = [np.float16, np.float32, np.float64, np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint16, np.uint32, np.uint64, np.bool_]


def _values(rng, dt, shape):
    if np.dtype(dt).kind == "f":
        return rng.standard_normal(shape).astype(dt)
    if dt is np.bool_:
        return rng.integers(0, 2, shape).astype(np.bool_)
    info = np.iinfo(dt)
    return rng.integers(info.min, info.max, shape, dtype=dt, endpoint=True)


def _struct(d, name="m", version=1, grpc_frame=False):
    n, preps = _example_columns(d)
    feats = (N.Feature * max(len(preps), 1))(*[p[0] for p in preps])
    rg = (N.Ragged * max(len(preps), 1))(*[p[3] or N.Ragged() for p in preps])
    nb = name.encode()
    req = N.ExampleRequest(model_name=nb, model_name_len=len(nb), has_version=int(version is not None), order=N.ORDER_UPB,
                           version=version or 0, n_examples=n, n_features=len(preps), flags=N.RF_GRPC_FRAME if grpc_frame else 0,
                           features=feats)
    return req, rg, (preps, feats, nb)


def _target(key):
    kb = key.encode() if isinstance(key, str) else key
    return N.ExampleTarget(kind=N.EXAMPLES_PREDICT_STRING, key=kb, key_len=len(kb))


def test_target_mirror():
    assert C.sizeof(N.ExampleTarget) == 24
    assert [f[0] for f in N.ExampleTarget._fields_] == ["kind", "pad_", "key", "key_len"]
    assert N.ExampleTarget.key.offset == 8 and N.ExampleTarget.key_len.offset == 16


@pytest.mark.parametrize("n", [0, 1, 127, 128, 16383, 16384])
def test_size_is_the_runtime_byte_size(n):
    rng = np.random.default_rng(n)
    lib = N.load()
    for t, key in enumerate(KEYS):
        width = 1 if n > 200 else int(rng.integers(0, 40))
        d = {"x": rng.standard_normal((n, width)).astype(rng.choice([np.float32, np.float64, np.float16]))}
        if t % 2:
            d["bias"] = np.float32(0.5)
            d["k" * (t * 30)] = rng.standard_normal((n, 2)).astype(np.float32)
        name, version = ("model", t) if t % 3 else ("", None)
        ref = predict_examples_request(name, version, d, key).ByteSize()
        for grpc_frame in (False, True):
            req, _, keep = _struct(d, name, version, grpc_frame)
            tg = _target(key)
            size = C.c_uint64()
            N.check(lib.b200tfs_example_target_request_size(C.byref(req), C.byref(tg), C.byref(size)))
            assert size.value == ref + (5 if grpc_frame else 0), (key, grpc_frame)
            # a LIST target, and no target at all, are the Classify size
            list_size, plain = C.c_uint64(), C.c_uint64()
            N.check(lib.b200tfs_example_target_request_size(C.byref(req), C.byref(N.ExampleTarget()), C.byref(list_size)))
            N.check(lib.b200tfs_example_request_size(C.byref(req), C.byref(plain)))
            assert list_size.value == plain.value


@pytest.mark.parametrize("seed", range(16))
def test_arena_bounds_requests_with_integer_and_ragged_columns(seed):
    rng = np.random.default_rng(100 + seed)
    n = int(rng.choice([0, 1, 9, 200]))
    d = {}
    for k in rng.choice(["a", "ab", "ids", "été"], size=int(rng.integers(1, 4)), replace=False):
        dt = ALL[int(rng.integers(len(ALL)))]
        if seed % 2:
            L = int(rng.choice([0, 1, 5, 40]))
            d[str(k)] = RaggedColumn(_values(rng, dt, (n, L)), rng.integers(0, L + 1, n))
        else:
            d[str(k)] = _values(rng, dt, (n, int(rng.integers(0, 6))))
    d["neg"] = np.full((n, 6), -1, np.int64)                 # ten bytes per element: the worst case
    keys = [KEYS[seed % len(KEYS)], "examples"]
    reqs, targets, keep = [], [], []
    for key in keys:
        req, rg, k = _struct(d, grpc_frame=bool(seed % 3))
        reqs.append(req)
        targets.append(_target(key))
        keep.append(k)
    ra, ta = (N.ExampleRequest * 2)(*reqs), (N.ExampleTarget * 2)(*targets)
    arena = C.c_uint64()
    N.check(N.load().b200tfs_example_target_arena_size(2, ra, ta, C.byref(arena)))
    need = sum(len(predict_examples_ref("m", 1, d, key, grpc_frame=bool(seed % 3))) for key in keys)
    assert arena.value >= need
    one = C.c_uint64()
    N.check(N.load().b200tfs_example_target_arena_size(1, ra, ta, C.byref(one)))
    assert one.value >= len(predict_examples_ref("m", 1, d, keys[0], grpc_frame=bool(seed % 3)))


def _refusals(req, tg):
    """every target entry point's status with no context: the size, the arena bound, _host and _async"""
    lib = N.load()
    out = C.c_uint64()
    off, ln = (C.c_uint64 * 1)(), (C.c_uint64 * 1)()
    buf = C.create_string_buffer(16)
    return [lib.b200tfs_example_target_request_size(C.byref(req), C.byref(tg), C.byref(out)),
            lib.b200tfs_example_target_arena_size(1, C.byref(req), C.byref(tg), C.byref(out)),
            lib.b200tfs_encode_example_targets_host(None, 1, C.byref(req), None, C.byref(tg), buf, 16, off, ln),
            lib.b200tfs_encode_example_targets_async(None, 1, C.byref(req), None, C.byref(tg), buf, 16)]


def test_target_refusals():
    req, _, keep = _struct({"x": np.zeros((4, 3), np.float32)})
    ok = _refusals(req, _target("examples"))
    assert ok == [N.OK, N.OK, N.E_ARG, N.E_ARG]              # well-formed: only the context is missing
    for kind in (2, -1, 0x100):
        tg = _target("examples")
        tg.kind = kind
        assert _refusals(req, tg) == [N.E_ARG] * 4 and "kind" in N.last_error()
    tg = _target("examples")
    tg.key_len = -1
    assert _refusals(req, tg) == [N.E_ARG] * 4
    tg = N.ExampleTarget(kind=N.EXAMPLES_PREDICT_STRING, key=None, key_len=3)
    assert _refusals(req, tg) == [N.E_ARG] * 4
    tg = N.ExampleTarget(kind=N.EXAMPLES_PREDICT_STRING, key=None, key_len=0)     # the empty key
    assert _refusals(req, tg)[:2] == [N.OK, N.OK]
    tg = _target("examples")
    tg.key_len = 1 << 31                                      # never read: refused by its length
    assert _refusals(req, tg) == [N.E_TOOBIG] * 4
    # the existing checks hold for a Predict target too
    empty, _, keep2 = _struct({"x": np.zeros((4, 0), np.float32)})
    empty.n_features = 0
    assert _refusals(empty, _target("examples"))[:3] == [N.E_ARG] * 3
    out = C.c_uint64()
    tg = _target("examples")
    assert N.load().b200tfs_example_target_request_size(C.byref(empty), C.byref(tg), C.byref(out)) == N.E_ARG
    assert "feature" in N.last_error()
    rreq, rg, keep3 = _struct({"r": RaggedColumn(np.zeros((4, 6), np.float32), [0, 1, 6, 2])})
    rg[0].unit = 2                                            # row_elems 6 != max_len 6 * unit 2
    off, ln = (C.c_uint64 * 1)(), (C.c_uint64 * 1)()
    buf = C.create_string_buffer(16)
    tg = _target("examples")
    assert N.load().b200tfs_encode_example_targets_host(None, 1, C.byref(rreq), rg, C.byref(tg), buf, 16, off, ln) == N.E_ARG
    rg[0].unit = 1
    bad = np.array([0, 7, 1, 1], np.int64)
    rg[0].lengths = bad.ctypes.data                           # past max_len: refused before any launch
    assert N.load().b200tfs_encode_example_targets_host(None, 1, C.byref(rreq), rg, C.byref(tg), buf, 16, off, ln) == N.E_SHAPE


@pytest.mark.parametrize("grpc_frame", [False, True])
def test_host_route_for_a_str_column(grpc_frame):
    d = {"s": np.array([["a", "été"], ["", "x"], ["y", "z"]]), "v": np.arange(3), "f": np.float32(2.5)}
    for key in ("examples", "", "中"):
        got = _host_example_request("m", 3, d, grpc_frame, key)
        assert got == predict_examples_ref("m", 3, d, key, grpc_frame=grpc_frame)
        assert _host_example_request("m", None, d, grpc_frame, key.encode()) == predict_examples_ref("m", None, d, key, grpc_frame=grpc_frame)
    assert _example_columns(d) is None                         # the device route does not take it
    assert _host_example_request("m", 3, d, grpc_frame) != _host_example_request("m", 3, d, grpc_frame, "examples")
