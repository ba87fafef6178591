"""Codec.encode_predict_requests_padded and b200tfs_encode_padded_requests_async: n PredictRequests cut out of one padded tensor per
input on the device, bit for bit against the definition - each request's boxes sliced on the host and encoded by
encode_predict_requests - and, for a few, against the reference's own serialisation through the oracle."""
import ctypes as C

import numpy as np
import pytest

from devutil import Dev, tensor_struct
from min_tfs_client import _native as N
from oracle import wire_oracle as O

pytestmark = pytest.mark.gpu


def _definition(codec, inputs, shapes, broadcast=None, model_version=3, **kw):
    n = len(next(iter(shapes.values())))
    S = {k: np.asarray(s, np.int64).reshape(n, -1) for k, s in shapes.items()}
    r0 = {k: np.concatenate([[0], np.cumsum(s[:, 0])]) for k, s in S.items()}
    reqs = []
    for r in range(n):
        d = {k: p[(slice(int(r0[k][r]), int(r0[k][r] + S[k][r][0])),) + tuple(slice(0, int(x)) for x in S[k][r][1:])]
             for k, p in inputs.items()}
        d.update(broadcast or {})
        reqs.append(("model", model_version, d))
    return codec.encode_predict_requests(reqs, **kw)


def _check(codec, inputs, shapes, broadcast=None, device=True, **kw):
    calls = codec.padded_encode_device_calls
    got = codec.encode_predict_requests_padded("model", inputs, shapes, model_version=3, broadcast=broadcast, **kw)
    got_bytes = [bytes(g) for g in got]
    want = _definition(codec, inputs, shapes, broadcast, **{k: v for k, v in kw.items() if k != "out"})
    assert got_bytes == want
    assert codec.padded_encode_device_calls == calls + (1 if device else 0)
    return got


def _ragged_rows(rng, n, R, m, dims):
    rows = rng.multinomial(R - rng.integers(0, R // 4 + 1), np.ones(n) / n)
    s = np.zeros((n, m), np.int64)
    s[:, 0] = rows
    for d in range(1, m):
        s[:, d] = rng.integers(0, dims[d] + 1, n)
    return s


_DT = [np.float32, np.float64, np.float16, np.complex64, np.complex128, np.bool_, np.int8, np.int16, np.int32, np.int64, np.uint8,
       np.uint16, np.uint32, np.uint64]


def _values(rng, shape, dt):
    dt = np.dtype(dt)
    if dt.kind == "b":
        return rng.integers(0, 4, shape).astype(np.uint8).view(np.bool_)     # bool bytes 2 and 3 too
    if dt.kind in "iu":
        info = np.iinfo(dt)
        return rng.integers(info.min, info.max, shape, dtype=dt, endpoint=True)
    a = (rng.standard_normal(shape) * 1e3).astype(dt)
    if dt == np.float32 and a.size >= 4:
        a.reshape(-1)[:4] = np.array([0x7F800001, 0xFF800001, 0x7FC00001, 0x80000000], np.uint32).view(np.float32)
    return a


@pytest.mark.parametrize("dt", _DT, ids=lambda d: np.dtype(d).name)
@pytest.mark.parametrize("full", [False, True], ids=["split", "boxes"])
def test_every_dtype(codec, dt, full):
    rng = np.random.default_rng(_DT.index(dt) + 100 * full)
    P = _values(rng, (40, 6, 5), dt)
    S = _ragged_rows(rng, 7, 40, 3, P.shape)
    _check(codec, {"x": P}, {"x": S if full else S[:, 0]})


@pytest.mark.parametrize("opts", [dict(keep_snan=True), dict(tensor_content=True), dict(wire_dtype="DT_FLOAT"), dict(grpc_frame=True),
                                  dict(order="given")], ids=lambda o: next(iter(o)))
def test_options(codec, opts):
    rng = np.random.default_rng(5)
    dt = np.float16 if "wire_dtype" in opts else np.float32
    P = _values(rng, (30, 9, 4), dt)
    S = _ragged_rows(rng, 5, 30, 3, P.shape)
    ids = rng.integers(-10 ** 6, 10 ** 6, (30, 9))
    bc = {} if "wire_dtype" in opts else {"first_ids": ids[:1, :2]}
    inputs = {"zz": P} if "wire_dtype" in opts else {"zz": P, "ids": ids}
    shapes = {"zz": S} if "wire_dtype" in opts else {"zz": S, "ids": S[:, :2]}
    _check(codec, inputs, shapes, broadcast=bc or None, **opts)


def test_rank4_ragged_hw_gather_and_rank3(codec):
    rng = np.random.default_rng(7)
    img = rng.standard_normal((6, 20, 24, 3)).astype(np.float32)
    S = np.array([[1, rng.integers(0, 21), rng.integers(0, 25), 3] for _ in range(6)], np.int64)
    _check(codec, {"image": img}, {"image": S})
    seq = rng.standard_normal((12, 16, 8)).astype(np.float64)
    S3 = np.array([[2, 16, 3], [3, 5, 8], [1, 0, 8], [4, 7, 2], [2, 16, 8]], np.int64)   # trimmed last axis, trimmed middle axis
    _check(codec, {"seq": seq}, {"seq": S3})
    ids = rng.integers(-(2 ** 63), 2 ** 63 - 1, (6, 20, 24), dtype=np.int64)
    _check(codec, {"ids": ids}, {"ids": S[:, :3]})


def test_batch_sizes_and_keys(codec):
    rng = np.random.default_rng(9)
    ids = rng.integers(0, 50000, (4096, 64))
    mask = np.ones((4096, 64), np.int64)
    S = np.stack([np.ones(4096, np.int64), rng.integers(1, 65, 4096)], 1)
    _check(codec, {"input_ids": ids, "attention_mask": mask}, {"input_ids": S, "attention_mask": S})
    _check(codec, {"input_ids": ids[:1]}, {"input_ids": S[:1]})
    eight = {f"k{i}": _values(rng, (20, 3), _DT[i]) for i in range(8)}
    sh = {k: _ragged_rows(rng, 4, 20, 2, (20, 3)) for k in eight}
    _check(codec, eight, sh, broadcast={"b0": np.float32(1.5), "b1": np.arange(3, dtype=np.int32)})
    nine = dict(eight, k8=_values(rng, (20, 3), np.int64))
    sh9 = dict(sh, k8=sh["k0"])
    _check(codec, nine, sh9, device=False)


def test_varint_boxes_over_one_counter_group(codec):
    # packed-varint boxes of more than 256 tiles (2048 elements each) in two inputs and several requests: every job's tile counters
    # are summed in groups of 256, and the groups of different jobs must stay apart
    rng = np.random.default_rng(21)
    ids = rng.integers(-(2 ** 40), 2 ** 40, (262144, 16))
    mask = rng.integers(0, 2, (262144, 16))
    _check(codec, {"input_ids": ids, "attention_mask": mask}, {"input_ids": np.full(4, 65536), "attention_mask": np.full(4, 65536)})
    S = np.array([[40000, 16], [90000, 9], [1, 16], [132143, 13]], np.int64)
    _check(codec, {"input_ids": ids, "attention_mask": mask}, {"input_ids": S, "attention_mask": S}, broadcast={"b": ids[:40000, 0]})


def test_sources_pinned_torch_and_misaligned(codec):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(11)
    P = rng.standard_normal((33, 17)).astype(np.float32)
    S = _ragged_rows(rng, 6, 33, 2, P.shape)
    pin = codec.pinned_empty(P.shape, np.float32)
    pin[...] = P
    got = _check(codec, {"x": pin}, {"x": S}, out="pinned")
    assert all(isinstance(g, np.ndarray) for g in got)
    big = torch.from_numpy(np.concatenate([np.zeros(1, np.float32), P.reshape(-1)])).cuda()
    tp = big[1:].view(33, 17)                                # 4 bytes past a 16-byte boundary
    ts = torch.from_numpy(S).cuda()
    torch.cuda.synchronize()
    calls = codec.padded_encode_device_calls
    got = codec.encode_predict_requests_padded("model", {"x": tp}, {"x": ts}, model_version=3)
    assert got == _definition(codec, {"x": P}, {"x": S})
    assert codec.padded_encode_device_calls == calls + 1
    i8 = torch.from_numpy(np.arange(1, 1 + 33 * 17 + 3, dtype=np.int8)).cuda()[3:].view(33, 17)
    torch.cuda.synchronize()
    got = codec.encode_predict_requests_padded("model", {"x": i8}, {"x": S}, model_version=3)
    assert got == _definition(codec, {"x": i8.cpu().numpy()}, {"x": S})


def test_against_the_oracle(codec):
    rng = np.random.default_rng(13)
    P = rng.standard_normal((10, 4, 3)).astype(np.float32)
    ids = rng.integers(-100, 100, (10, 4))
    S = np.array([[3, 2, 3], [0, 4, 1], [5, 4, 3]], np.int64)
    got = codec.encode_predict_requests_padded("m", {"x": P, "ids": ids}, {"x": S, "ids": S[:, :2]}, model_version=1,
                                               broadcast={"t": np.float32(2.0)})
    r0 = 0
    for r in range(3):
        x = P[r0:r0 + S[r, 0], :S[r, 1], :S[r, 2]]
        i = ids[r0:r0 + S[r, 0], :S[r, 1]]
        r0 += S[r, 0]
        assert got[r] == O.encode_predict_request("m", 1, [("x", x), ("ids", i), ("t", np.float32(2.0))], order="upb")


def test_host_shape_errors(codec):
    P = np.zeros((5, 3), np.float32)
    for bad in (np.array([[2, 4]]), np.array([[-1, 3]]), np.array([[3, 3], [3, 3]]), np.zeros((2, 3), np.int64), np.zeros((1, 1, 2), np.int64)):
        with pytest.raises(ValueError):
            codec.encode_predict_requests_padded("m", {"x": P}, {"x": bad})
    with pytest.raises(ValueError):
        codec.encode_predict_requests_padded("m", {"x": P, "y": P}, {"x": np.array([1, 1]), "y": np.array([1])})


def _abi_request(dev, arrays, shapes_dev, bcast=()):
    structs, keep, pins = [], [], []
    for k, (ptr, a) in arrays.items():
        t, dims = tensor_struct(ptr, a, key=k.encode(), flags=N.F_BROADCAST if k in bcast else 0)
        keep.append(dims)
        structs.append(t)
        if k in bcast:
            pins.append(N.PadInput(shapes=None, cols=0))
        else:
            sp, cols = shapes_dev[k]
            pins.append(N.PadInput(shapes=sp, cols=cols))
    arr = (N.Tensor * len(structs))(*structs)
    name = b"model"
    req = N.Request(model_name=name, model_name_len=len(name), has_version=1, order=N.ORDER_UPB, version=3, n_inputs=len(structs),
                    flags=0, inputs=arr)
    return req, (N.PadInput * len(pins))(*pins), (keep, arr, name)


def test_graph_replay_statuses_and_canaries(codec):
    dev = Dev()
    try:
        rng = np.random.default_rng(17)
        n, R = 64, 256
        P = rng.standard_normal((R, 32, 4)).astype(np.float32)
        ids = rng.integers(0, 50000, (R, 32))
        S = _ragged_rows(rng, n, R, 3, P.shape)
        pP, pI = dev.upload(P), dev.upload(ids)
        pS, pS2 = dev.upload(S), dev.upload(np.ascontiguousarray(S[:, :2]))
        req, pins, keep = _abi_request(dev, {"x": (pP, P), "ids": (pI, ids)}, {"x": (pS, 3), "ids": (pS2, 2)})
        cap = C.c_uint64()
        N.check(dev.lib.b200tfs_padded_request_arena_size(n, C.byref(req), C.byref(cap)))
        base = dev.malloc(cap.value + 512)
        arena = (base + 255) & ~255
        canary = np.full(cap.value + 256, 0xA5, np.uint8)

        def run(graph=None):
            N.check(dev.lib.b200tfs_memcpy_h2d(dev.ctx, arena, canary.ctypes.data, canary.size))
            if graph is None:
                N.check(dev.lib.b200tfs_encode_padded_requests_async(dev.ctx, n, C.byref(req), pins, arena, cap.value))
            else:
                N.check(dev.lib.b200tfs_graph_launch(dev.ctx, graph))
            off, ln = (C.c_uint64 * n)(), (C.c_uint64 * n)()
            rc = dev.lib.b200tfs_encode_results(dev.ctx, n, off, ln)
            wire = dev.download(arena, canary.size)
            return rc, [int(o) for o in off], [int(x) for x in ln], wire

        def expect(P, ids, S):
            return _definition(codec, {"x": P, "ids": ids}, {"x": S, "ids": S[:, :2]})

        def verify(res, want):
            rc, off, ln, wire = res
            assert rc == N.OK
            used = np.zeros(wire.size, bool)
            for r in range(n):
                assert wire[off[r]: off[r] + ln[r]].tobytes() == want[r]
                used[off[r]: off[r] + ln[r]] = True
            assert (wire[~used] == 0xA5).all()              # between records, around the arena
            assert all(off[r] + ln[r] <= off[r + 1] for r in range(n - 1))

        verify(run(), expect(P, ids, S))
        N.check(dev.lib.b200tfs_capture_begin(dev.ctx))
        N.check(dev.lib.b200tfs_encode_padded_requests_async(dev.ctx, n, C.byref(req), pins, arena, cap.value))
        g = C.c_void_p()
        N.check(dev.lib.b200tfs_capture_end(dev.ctx, C.byref(g)))
        # new shapes and values into the same buffers, then replay
        P2 = rng.standard_normal(P.shape).astype(np.float32)
        ids2 = rng.integers(-(2 ** 40), 2 ** 40, ids.shape)
        S_new = _ragged_rows(rng, n, R, 3, P.shape)
        for ptr, a in ((pP, P2), (pI, ids2), (pS, S_new), (pS2, np.ascontiguousarray(S_new[:, :2]))):
            N.check(dev.lib.b200tfs_memcpy_h2d(dev.ctx, ptr, a.ctypes.data, a.nbytes))
        verify(run(g.value), expect(P2, ids2, S_new))
        # invalid device shapes: a negative dim (E_SHAPE) and rows past R (E_SIZE, that request and every later one)
        S_bad = S_new.copy()
        S_bad[3, 2] = -1
        S_bad[40, 0] = R
        for ptr, a in ((pS, S_bad), (pS2, np.ascontiguousarray(S_bad[:, :2]))):
            N.check(dev.lib.b200tfs_memcpy_h2d(dev.ctx, ptr, a.ctypes.data, a.nbytes))
        rc, off, ln, wire = run(g.value)
        assert rc == N.E_SHAPE
        assert ln[3] == 0 and all(ln[r] == 0 for r in range(40, n)) and all(ln[r] > 0 for r in range(40) if r != 3)
        want = expect(P2, ids2, np.where(np.arange(n)[:, None] == 3, S_new, S_bad)[:40])
        used = np.zeros(wire.size, bool)
        for r in range(40):
            if r != 3:
                assert wire[off[r]: off[r] + ln[r]].tobytes() == want[r]
                used[off[r]: off[r] + ln[r]] = True
        assert (wire[~used] == 0xA5).all()
        N.check(dev.lib.b200tfs_graph_destroy(g.value))
    finally:
        dev.close()
