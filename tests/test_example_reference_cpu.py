"""The tf.Example request reference and geometry model of example_ref.py, pinned without a GPU: the bytes against the protobuf
runtime (ragged_ref, predict_examples_ref), the model's constants and slot placement against the sources and
b200tfs_example_target_arena_size, and the emit model's invariants - every byte stored exactly once, and the in-place path's
flush of earlier bytes unreachable under today's host planning."""
import ctypes as C

import numpy as np
import pytest

import cast_sweep as CS
import example_ref as R
from min_tfs_client import _native as N
from min_tfs_client.codec import RaggedColumn, _example_columns
from min_tfs_client.requests import TensorServingClient
from predict_examples_ref import predict_examples_ref
from ragged_ref import ragged_ref
from tensorflow_serving.apis.classification_pb2 import ClassificationRequest

ALL = [np.float16, np.float32, np.float64, np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint16, np.uint32, np.uint64, np.bool_]


def _values(rng, dt, shape):
    if np.dtype(dt).kind == "f":
        return rng.standard_normal(shape).astype(dt)
    if dt is np.bool_:
        return rng.integers(0, 2, shape).astype(np.bool_)
    info = np.iinfo(dt)
    return rng.integers(info.min, info.max, shape, dtype=dt, endpoint=True)


def _same(d, name="m", version=1, grpc=False):
    """the reference equals the runtime, as an example_list and as a Predict request"""
    if any(isinstance(v, RaggedColumn) for v in d.values()):
        ref = ragged_ref(name, version, d, grpc_frame=grpc)
    else:
        ref = TensorServingClient._make_example_request(None, ClassificationRequest, name, d, version).SerializeToString(deterministic=True)
        ref = (b"\x00" + len(ref).to_bytes(4, "big") + ref) if grpc else ref
    assert R.request_bytes(name, version, d, grpc=grpc) == ref
    for key in ("examples", "", "中"):
        assert R.request_bytes(name, version, d, key=key, grpc=grpc) == predict_examples_ref(name, version, d, key, grpc_frame=grpc)


def _f64_sweep():
    rng = np.random.default_rng(5)
    vals = [(e << 52) | m for e in range(0, 2048, 3) for m in (0x10000000, 0x10000001, 0x0FFFFFFF, 0xFFFFFFFFFFFFF, 0)]
    vals += [0x47EFFFFFF0000000, 0x3690000000000001, 0x7FF0000000000001, 0x7FF4000020000000, 0x7FF000001FFFFFFF]
    vals += [int(v) for v in rng.integers(0, 1 << 63, 500, dtype=np.uint64)]
    bits = np.array(vals, dtype=np.uint64)
    bits = np.concatenate([bits, bits | np.uint64(1 << 63)])
    return np.concatenate([bits, np.zeros((-len(bits)) % 64, np.uint64)]).view(np.float64).reshape(-1, 64)


@pytest.mark.parametrize("dt", ALL, ids=lambda t: np.dtype(t).name)
def test_every_dtype(dt):
    x = _values(np.random.default_rng(1), dt, (20, 3))
    _same({"v": x, "w": x[:, 0].copy(), "s": x[0, 0], "r": RaggedColumn(x, np.arange(20) % 4)})


def test_float_sweeps():
    f32 = CS.f32_patterns()
    _same({"f": np.concatenate([f32, np.zeros((-len(f32)) % 1024, np.uint32)]).view(np.float32).reshape(-1, 1024)})
    _same({"h": CS.all_f16().reshape(-1, 256)})
    with np.errstate(all="ignore"):
        _same({"d": _f64_sweep()})


def test_integer_extremes_and_bool_bytes():
    v = np.array([(1 << (7 * k)) - 1 for k in range(1, 10)] + [1 << 62, -1, -(1 << 63), (1 << 63) - 1, 0], dtype=np.int64)
    _same({"i": v.reshape(1, -1), "j": v[::-1].reshape(1, -1)})
    _same({"u": np.array([0, 1, 1 << 63, (1 << 63) + 5, (1 << 64) - 1, 127, 128], dtype=np.uint64).reshape(-1, 1)})
    for dt in ALL[3:11]:
        info = np.iinfo(dt)
        _same({"x": np.array([info.min, info.max, 0, -1 if info.min else 1], dtype=dt).reshape(2, 2)})
    _same({"b": np.frombuffer(bytes([2, 0, 1, 255, 0, 7]), dtype=np.bool_).reshape(3, 2)})


def test_shapes():
    _same({})
    _same({"a": np.float32(3.0), "b": np.int64(-4)}, version=None)                          # all 0-d: one example
    _same({"a": np.zeros((0, 4), np.float32), "b": np.zeros((0,), np.int64)}, name="")      # n = 0
    _same({"a": np.zeros((5, 0), np.float32), "b": np.zeros((5, 0), np.int32), "c": np.ones(5, np.int8)}, version=0, grpc=True)
    rng = np.random.default_rng(2)
    _same({"u0": RaggedColumn(np.zeros((6, 4, 0), np.int64), [0, 4, 1, 2, 3, 0]),                # unit 0
           "u3": RaggedColumn(rng.standard_normal((6, 4, 3)).astype(np.float16), [0, 4, 1, 2, 3, 0]),
           "i3": RaggedColumn(rng.integers(-9, 9, (6, 2, 3)).astype(np.int8), [2, 0, 1, 2, 1, 0])}, version=7)


def test_keys():
    rng = np.random.default_rng(3)
    keys = ["", "é", "中", "a", "ab", "abc", "b", "k" * 127, "l" * 128, "m" * 16384]
    d = {k: rng.integers(-5, 5, (3, 2)) if i % 2 else rng.standard_normal((3, 1)).astype(np.float32) for i, k in enumerate(keys)}
    _same(d, name="n" * 128, version=1 << 40)


@pytest.mark.parametrize("n_feat", [33, 200])
def test_many_features(n_feat):
    for rot in range(len(R.KINDS)):
        _same(R.chunk_case(n_feat, rot, n=6, seed=rot), grpc=rot == 2)


def test_given_order():
    d = {"zz": np.arange(6, dtype=np.float32).reshape(3, 2), "a": np.arange(3), "ab": np.ones(3, np.float64)}
    got, det = R.request_bytes("m", 2, d, order="given"), R.request_bytes("m", 2, d)
    assert got != det and ClassificationRequest.FromString(got) == ClassificationRequest.FromString(det)
    pos = [got.find(k.encode()) for k in d]
    assert pos == sorted(pos)
    ordered = {k: d[k] for k in ("ab", "a", "zz")}                   # already in the runtime's order
    assert R.request_bytes("m", 2, ordered, order="given") == det


def test_edge_cases_small():
    """small versions of the GPU edge cases"""
    d, want = R.nested_case((127, 128))
    _same(d)
    n, cols = R.columns(d)
    L = R.nested(cols, n)
    assert all((L[q][0, i] if L[q].ndim == 2 else L[q][i]) == t for i, (q, t) in enumerate(want))
    for S, n in ((5459, 9), (16377, 3), (16401, 2), (100, 3)):
        d = R.fixed_size(S, n)
        assert R.example_bytes(d)[0].tolist() == [S] * n
        _same(d)
    _same({"": RaggedColumn(np.ones((8, 1000), np.int64), np.arange(8) % 2)})
    for q in ("inner", "outer"):
        for t in (127, 128, 16383, 16384):
            for key in (None, "e"):
                d = R.request_case(q, t, key)
                _same(d)
                S = R.example_bytes(d)[0]
                assert R.request_lengths(R.ReqPlan("m", 1, d, key), int(S.sum()), key)[q] == t
    _same(R.counted_case(40), grpc=True)


# ---- the model against the sources ------------------------------------------------------------------------------------------
def test_constants_match_sources():
    assert (R.K_STAGE, R.K_EMIT_THREADS, R.K_TILE) == (16384, 256, R.K_PLAN_THREADS)
    k = R._source("example_kernels.cuh")
    assert "img[kExStage + 16]" in k and "for (uint32_t c = 0; c < q.n_feat; c += 32)" in k
    assert "for (uint32_t k0 = q.first_tile; k0 < t; k0 += kExTile)" in k
    assert "for (uint32_t k = lane; k < q.n_tiles; k += 32)" in k
    h = R._source("example_host.inc")
    assert "std::max<uint64_t>(1, kExStage / X.ex_max)" in h and "e0 += kExTile" in h


def _structs(items):
    keep, structs, tg = [], [], []
    for name, version, d, key, grpc in items:
        n, preps = _example_columns(d)
        feats = (N.Feature * max(len(preps), 1))(*[p[0] for p in preps])
        nb = name.encode()
        structs.append(N.ExampleRequest(model_name=nb, model_name_len=len(nb), has_version=int(version is not None), order=N.ORDER_UPB,
                                        version=version or 0, n_examples=n, n_features=len(preps), flags=N.RF_GRPC_FRAME if grpc else 0,
                                        features=feats))
        kb = key.encode() if key is not None else None
        tg.append(N.ExampleTarget(kind=N.EXAMPLES_PREDICT_STRING, key=kb, key_len=len(kb)) if kb is not None else N.ExampleTarget())
        keep.append((preps, feats, nb, kb))
    return (N.ExampleRequest * len(structs))(*structs), (N.ExampleTarget * len(tg))(*tg), keep


def _random_request(rng, n):
    d = {}
    for k in range(int(rng.integers(1, 5))):
        dt = ALL[int(rng.integers(len(ALL)))]
        w = int(rng.choice([0, 1, 7, 300, 5000]))
        v = np.broadcast_to(np.zeros(1, dt), (n, w))
        d["k" * int(rng.integers(0, 200)) + str(k)] = RaggedColumn(v, np.zeros(n, np.int64)) if rng.random() < 0.3 else v
    return d


@pytest.mark.parametrize("seed", range(12))
def test_slot_placement_matches_arena_size(seed):
    rng = np.random.default_rng(seed)
    items = []
    for r in range(int(rng.integers(1, 6))):
        key = [None, "examples", "k" * 200][r % 3]
        items.append(("m" * int(rng.integers(0, 300)), [None, 0, 1 << 40][r % 3], _random_request(rng, int(rng.integers(0, 3000))), key,
                      bool(rng.integers(2))))
    reqs, tg, keep = _structs(items)
    cap = C.c_uint64()
    plans = []
    for k in range(len(items)):          # every prefix of the call: the slot end of its last request
        N.check(N.load().b200tfs_example_target_arena_size(k + 1, reqs, tg, C.byref(cap)))
        plans.append(R.ReqPlan(items[k][0], items[k][1], items[k][2], items[k][3], items[k][4]))
        assert R.plan(plans) == cap.value == plans[-1].slot_end
    for q in plans:
        assert q.anchor % 16 == 0 and q.slot_off % 256 == 0 and q.anchor - q.slot_off >= q.prefix_max


def test_shortest_examples_bound_the_count():
    """the host refuses exactly the requests whose examples at their shortest (one byte per integer element) exceed 2 GiB"""
    d = {"a": np.zeros((1, 100), np.int8), "b": np.zeros((1, 1), np.int16)}
    q = R.ReqPlan("m", 1, d)
    reqs, tg, keep = _structs([("m", 1, d, None, False)])
    cap = C.c_uint64()
    for n, rc in ((R.PROTO_LIMIT // q.ex_min, N.OK), (R.PROTO_LIMIT // q.ex_min + 1, N.E_TOOBIG)):
        reqs[0].n_examples = n
        assert N.load().b200tfs_example_target_arena_size(1, reqs, tg, C.byref(cap)) == rc
    assert q.ex_min == R.example_bytes({"a": np.zeros((1, 100), np.int8), "b": np.zeros((1, 1), np.int16)})[0][0]
    assert q.ex_max == R.example_bytes({"a": np.full((1, 100), -1, np.int8), "b": np.full((1, 1), -1, np.int16)})[0][0]


# ---- the emit model's invariants ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(40))
def test_emit_model_covers_every_byte_once(seed):
    """Random plans and example sizes: the stores cover the examples exactly once, and an example written in place never has
    earlier bytes of its span to flush - with per >= 2 no example reaches the in-place path at all.  This is a property of
    today's host planning (spans of at most kExStage / ex_max examples at their longest); a planner that sizes spans from the
    real sizes makes the flush reachable and needs a GPU case for it."""
    rng = np.random.default_rng(seed)
    cursor_items = []
    for r in range(int(rng.integers(1, 4))):
        n = int(rng.integers(1, 400))
        w = int(rng.choice([1, 30, 1000, 2000, 4090, 4100, 8000]))
        counted = bool(rng.integers(2))
        v = np.broadcast_to(np.zeros(1, np.int8 if counted else np.float32), (n, w))
        q = R.ReqPlan("m", 1, {"k" * int(rng.integers(1, 30)): v}, "x" if r % 2 else None, bool(rng.integers(2)))
        cursor_items.append(q)
    R.plan(cursor_items)
    for q in cursor_items:
        sizes = rng.integers(q.ex_min, q.ex_max + 1, q.n) if q.counted else np.full(q.n, q.ex_max)
        m = R.emit(q, sizes)
        assert R.covers_once(q, sizes, m["stores"])
        assert all(flushed == 0 for _, _, flushed in m["in_place"])
        assert q.per == 1 or not m["in_place"]
        assert all(fill <= R.K_STAGE for _, _, _, fill, _ in m["batches"])
