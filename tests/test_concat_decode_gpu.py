"""Codec.decode_predict_responses_concat and b200tfs_decode_concat: a batch of PredictResponses decoded into one tensor per key,
concatenated along axis 0 on the device, against np.concatenate over the per-response decode."""
import ctypes as C

import numpy as np
import pytest

from min_tfs_client import _native as N
from oracle import wire_oracle as O

pytestmark = pytest.mark.gpu

DTYPES = [np.float32, np.float64, np.int32, np.int64, np.uint8, np.int8, np.int16, np.uint16, np.uint32, np.uint64, np.bool_,
          np.float16, np.complex64, np.complex128]


def _values(rng, dtype, shape):
    dt = np.dtype(dtype)
    if dt.kind == "b":
        return rng.integers(0, 2, shape).astype(np.bool_)
    if dt.kind in "iu":
        info = np.iinfo(dt)
        return rng.integers(info.min, info.max, shape, dtype=dt, endpoint=True)
    if dt.kind == "c":
        return (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).astype(dt)
    return rng.standard_normal(shape).astype(dt)


def _expect(codec, wires, keys, strict=False, out_dtypes=None, oracle=True):
    per = [codec.decode_predict_responses([w], strict=strict, out_dtypes=out_dtypes)[0] for w in wires]
    for w, (arrays, _) in zip(wires, per):   # the per-response decode itself agrees with the oracle
        ref = O.decode_predict_response(w, strict=strict) if oracle and out_dtypes is None else {}
        for k in ref:
            assert arrays[k].tobytes() == ref[k].tobytes()
    return {k: np.concatenate([p[0][k] for p in per], axis=0) for k in keys}


def _same(got, want):
    for k, w in want.items():
        g = got[k]
        if hasattr(g, "copy_to_host"):
            g = g.copy_to_host()
        assert g.dtype == w.dtype and g.shape == w.shape, k
        assert g.tobytes() == w.tobytes(), k


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: np.dtype(d).name)
@pytest.mark.parametrize("strict", [False, True])
def test_every_dtype_with_varying_rows(codec, dtype, strict):
    if strict and np.dtype(dtype).kind == "c":
        pytest.skip("strict decode rejects complex outputs")
    rng = np.random.default_rng(1)
    rows = [3, 0, 7, 1, 0, 12]
    wires = [O.build_predict_response([("y", _values(rng, dtype, (r, 5)))]) for r in rows]
    before = codec.concat_device_calls
    got, specs = codec.decode_predict_responses_concat(wires, ["y"], strict=strict)
    assert codec.concat_device_calls == before + 1          # the device route, not the response-by-response one
    _same(got, _expect(codec, wires, ["y"], strict))
    assert len(specs) == len(wires) and specs[0].name == "default"


@pytest.mark.parametrize("rank", [1, 2, 3, 4, 20])
def test_ranks(codec, rank):
    rng = np.random.default_rng(rank)
    tail = (2,) * (rank - 1) if rank == 20 else (3, 2, 4)[: rank - 1]
    wires = [O.build_predict_response([("x", rng.standard_normal((r,) + tail).astype(np.float32))]) for r in (2, 1, 3)]
    got, _ = codec.decode_predict_responses_concat(wires)
    _same(got, _expect(codec, wires, ["x"]))


def test_eight_keys_in_different_map_orders_and_a_single_record(codec):
    rng = np.random.default_rng(2)
    keys = [f"k{i}" for i in range(8)]
    wires = []
    for r in range(5):
        outs = [(k, _values(rng, DTYPES[i % 11], (r + i % 3, 2))) for i, k in enumerate(keys)]
        rng.shuffle(outs)
        wires.append(O.build_predict_response(outs))
    before = codec.concat_device_calls
    got, _ = codec.decode_predict_responses_concat(wires)
    assert codec.concat_device_calls == before + 1
    _same(got, _expect(codec, wires, keys))
    got, _ = codec.decode_predict_responses_concat(wires[:1], ["k3", "k0"])
    _same(got, _expect(codec, wires[:1], ["k3", "k0"]))


def test_4096_records_two_keys(codec):
    rng = np.random.default_rng(3)
    wires = [O.build_predict_response([("classes", rng.integers(0, 1000, (int(r), 5), dtype=np.int64)),
                                       ("scores", rng.standard_normal((int(r), 5)).astype(np.float32))])
             for r in rng.integers(0, 4, 4096)]
    before = codec.concat_device_calls
    got, specs = codec.decode_predict_responses_concat(wires)
    assert codec.concat_device_calls == before + 1
    _same(got, _expect(codec, wires, ["classes", "scores"]))
    assert len(specs) == 4096


@pytest.mark.parametrize("to", [np.float16, "bfloat16"])
def test_narrowing_casts(codec, to):
    from cast_sweep import f32_patterns

    if to == "bfloat16":
        from min_tfs_client.constants import BFLOAT16

        if BFLOAT16 is None:
            pytest.skip("needs ml_dtypes")
        to = BFLOAT16
    vals = f32_patterns().view(np.float32).ravel()[: 4096 * 3]
    parts = np.array_split(vals[: (vals.size // 4) * 4].reshape(-1, 4), 3)
    wires = [O.build_predict_response([("s", p), ("n", np.arange(p.shape[0], dtype=np.int64))]) for p in parts]
    before = codec.concat_device_calls
    got, _ = codec.decode_predict_responses_concat(wires, out_dtypes={"s": to})
    assert codec.concat_device_calls == before + 1
    _same(got, _expect(codec, wires, ["s", "n"], out_dtypes={"s": to}))


def test_device_result_out_and_pinned(codec):
    rng = np.random.default_rng(4)
    wires = [O.build_predict_response([("s", rng.standard_normal((r, 10)).astype(np.float32))]) for r in (4, 5, 6)]
    want = _expect(codec, wires, ["s"])
    got, _ = codec.decode_predict_responses_concat(wires, device=True)
    assert hasattr(got["s"], "__cuda_array_interface__")
    _same(got, want)
    pinned = codec.pinned_empty((15, 10), np.float32)
    got, _ = codec.decode_predict_responses_concat(wires, out={"s": pinned})
    assert got["s"] is pinned
    _same(got, want)
    torch = pytest.importorskip("torch")
    if torch.cuda.is_available():
        t = torch.empty((15, 10), dtype=torch.float32, device="cuda")
        got, _ = codec.decode_predict_responses_concat(wires, out={"s": t})
        torch.cuda.synchronize()
        assert t.cpu().numpy().tobytes() == want["s"].tobytes()
        assert torch.as_tensor(codec.decode_predict_responses_concat(wires, device=True)[0]["s"], device="cuda").cpu().numpy().tobytes() == \
            want["s"].tobytes()


def _raises_like(codec, wires, keys, **kw):
    try:
        _expect(codec, wires, keys, oracle=False, **{k: v for k, v in kw.items() if k in ("strict", "out_dtypes")})
        want = None
    except Exception as e:  # noqa: BLE001
        want = type(e)
    if want is None:
        codec.decode_predict_responses_concat(wires, keys, **kw)
        return None
    with pytest.raises(want):
        codec.decode_predict_responses_concat(wires, keys, **kw)
    return want


def test_error_classes(codec):
    f = lambda *s: np.ones(s, np.float32)  # noqa: E731
    good = O.build_predict_response([("a", f(2, 3))])
    assert _raises_like(codec, [good, O.build_predict_response([("b", f(2, 3))])], ["a"]) is KeyError
    assert _raises_like(codec, [good, O.build_predict_response([("a", f(2, 4))])], ["a"]) is ValueError
    assert _raises_like(codec, [good, O.build_predict_response([("a", f(2, 3, 1))])], ["a"]) is ValueError
    with pytest.raises(ValueError):
        codec.decode_predict_responses_concat([good, O.build_predict_response([("a", np.ones((2, 3), np.float64))])], ["a"])
    with pytest.raises(ValueError):
        codec.decode_predict_responses_concat([])
    assert _raises_like(codec, [good, good[:-3], O.build_predict_response([("b", f(1))])], ["a"]) is not None
    rank0 = O.build_predict_response([("a", np.float32(1.0))])
    _raises_like(codec, [good, rank0], ["a"])
    _raises_like(codec, [good, rank0], ["a"], strict=True)
    wide = O.build_predict_response([("a", np.array([300, 1], np.int64))])
    _raises_like(codec, [wide], ["a"])


def test_only_requested_outputs_are_decoded_on_either_route(codec):
    f = lambda *s: np.ones(s, np.float32)  # noqa: E731
    bad = O.build_predict_response([("a", f(2, 3)), ("b", np.ones(3, np.float32))])
    bad = bad.replace(b"\x12\x04\x12\x02\x08\x03", b"\x12\x04\x12\x02\x08\x04", 1)      # b: shape [4], three values
    with pytest.raises(ValueError):
        codec.decode_predict_responses([bad], strict=True)
    good = O.build_predict_response([("a", f(1, 3))])
    wide = O.build_predict_response([("a", f(1, 3))] + [(f"z{i}", f(1)) for i in range(9)])      # 10 outputs: response by response
    for wires in ([good, bad], [wide, bad]):
        before = codec.concat_device_calls
        got, _ = codec.decode_predict_responses_concat(wires, ["a"], strict=True, out_dtypes={"b": np.float16})
        assert codec.concat_device_calls == before + (1 if wires[0] is good else 0)
        assert got["a"].tobytes() == np.ones((3, 3), np.float32).tobytes()
        with pytest.raises(KeyError):
            codec.decode_predict_responses_concat(wires, ["a"], out={"b": np.empty(3, np.float32)})


# ---- C level -------------------------------------------------------------------------------------------------
def _c_batch(codec, wires, keys, fill=0xEE, caps=None):
    lib, ctx = codec._lib, codec.ctx
    buf, off, ln = codec._pack_wires(wires)
    n, nk = len(wires), len(keys)
    ck = (N.ConcatKey * nk)()
    kb = [k.encode() for k in keys]
    for i, k in enumerate(kb):
        ck[i].key, ck[i].key_len = k, len(k)
    N.check(lib.b200tfs_concat_layout(buf.ctypes.data, n, off, ln, nk, ck, 0))
    arena = codec.device_array(np.frombuffer(bytes(buf), np.uint8))
    dsts = []
    for i in range(nk):
        cap = int(ck[i].bytes) if caps is None else caps[i]
        d = codec.device_array(np.full(cap + 512, fill, np.uint8))
        dsts.append(d)
        ck[i].dst, ck[i].dst_cap = d.ptr, cap
    return lib, ctx, buf, off, ln, ck, kb, arena, dsts


def _results(codec, n, nk):
    outs, specs, st = (N.Output * (n * nk))(), (N.ModelSpec * n)(), (C.c_int32 * n)()
    N.check(codec._lib.b200tfs_concat_results(codec.ctx, n, nk, outs, specs, st))
    return outs, st


def test_c_route_is_all_ok_writes_only_its_ranges_and_counts_its_launches(codec):
    rng = np.random.default_rng(6)
    wires = [O.build_predict_response([("s", rng.standard_normal((r, 7)).astype(np.float32)),
                                       ("c", rng.integers(0, 1000, (r, 3), dtype=np.int64))]) for r in (3, 0, 5, 2)]
    keys = ["s", "c"]
    lib, ctx, buf, off, ln, ck, kb, arena, dsts = _c_batch(codec, wires, keys)
    before = codec.kernel_launches()
    N.check(lib.b200tfs_decode_concat(ctx, arena.ptr, len(wires), off, ln, 2, ck))
    outs, st = _results(codec, len(wires), 2)
    assert codec.kernel_launches() - before == 6
    assert all(st[r] == N.OK for r in range(len(wires)))
    assert all(outs[j].status == N.OK for j in range(len(wires) * 2))
    want = _expect(codec, wires, keys)
    for i, k in enumerate(keys):
        got = dsts[i].copy_to_host()
        nb = int(ck[i].bytes)
        assert got[:nb].tobytes() == want[k].tobytes()
        assert (got[nb:] == 0xEE).all()


def test_c_route_too_small_dst_cap_is_e_size_and_stores_nothing_past_it(codec):
    rng = np.random.default_rng(7)
    wires = [O.build_predict_response([("s", rng.standard_normal((4, 8)).astype(np.float32))]) for _ in range(3)]
    cap = 2 * 4 * 8 * 4 + 16           # room for two records and a bit
    lib, ctx, buf, off, ln, ck, kb, arena, dsts = _c_batch(codec, wires, ["s"], caps=[cap])
    N.check(lib.b200tfs_decode_concat(ctx, arena.ptr, 3, off, ln, 1, ck))
    outs, st = _results(codec, 3, 1)
    assert [outs[r].status for r in range(3)] == [N.OK, N.OK, N.E_SIZE]
    got = dsts[0].copy_to_host()
    assert (got[cap:] == 0xEE).all()
    assert got[:256].tobytes() == np.concatenate([O.decode_predict_response(w)["s"] for w in wires[:2]]).tobytes()


def test_c_graph_replay_adapts_to_new_row_counts(codec):
    # same record lengths, other row counts: int64 ids packed as varints of different byte lengths
    def rec(n_rows, big):
        ids = np.full((n_rows, 2), 300 if big else 1, np.int64)
        return O.build_predict_response([("ids", ids)])
    a2 = [rec(8, False), rec(4, True)]      # 16 B each
    b2 = [rec(4, True), rec(8, False)]      # the same lengths, rows swapped
    assert [len(w) for w in a2] == [len(w) for w in b2]
    from min_tfs_client.codec import Codec

    gc = Codec(0)           # a captured graph pins the context's scratch buffers: keep it off the shared codec
    lib, ctx, buf, off, ln, ck, kb, arena, dsts = _c_batch(gc, a2, ["ids"])
    N.check(lib.b200tfs_decode_concat(ctx, arena.ptr, 2, off, ln, 1, ck))
    _results(gc, 2, 1)
    N.check(lib.b200tfs_capture_begin(ctx))
    N.check(lib.b200tfs_decode_concat(ctx, arena.ptr, 2, off, ln, 1, ck))
    g = C.c_void_p()
    N.check(lib.b200tfs_capture_end(ctx, C.byref(g)))
    buf2, _, _ = gc._pack_wires(b2)
    N.check(lib.b200tfs_memcpy_h2d(ctx, arena.ptr, buf2.ctypes.data, buf2.nbytes))
    N.check(lib.b200tfs_graph_launch(ctx, g))
    outs, st = _results(gc, 2, 1)
    N.check(lib.b200tfs_graph_destroy(g))
    assert outs[0].status == N.OK and outs[1].status == N.OK and outs[1].dst_off == 4 * 2 * 8
    want = _expect(codec, b2, ["ids"])["ids"]
    assert dsts[0].copy_to_host()[: want.nbytes].tobytes() == want.tobytes()
    del arena, dsts
    gc.close()


def test_host_wire_form(codec):
    rng = np.random.default_rng(8)
    wires = [O.build_predict_response([("s", rng.standard_normal((r, 3)).astype(np.float32))]) for r in (1, 2)]
    lib, ctx, buf, off, ln, ck, kb, arena, dsts = _c_batch(codec, wires, ["s"])
    N.check(lib.b200tfs_decode_concat_host_async(ctx, buf.ctypes.data, 2, off, ln, 1, ck))
    outs, st = _results(codec, 2, 1)
    want = _expect(codec, wires, ["s"])["s"]
    assert dsts[0].copy_to_host()[: want.nbytes].tobytes() == want.tobytes()


_EXC_OF = {N.E_PARSE: ("DecodeError",), N.E_SHAPE: ("ValueError", "TypeError"), N.E_DTYPE: ("ValueError",), N.E_KEY: ("KeyError",),
           N.E_RANGE: ("OverflowError",)}


def _key_outcome(codec, w, key, ref):
    """What np.concatenate over the per-response decode (strict, the requested output only) does with record `w` next to the
    valid record `ref`: (exception name or None, the record's rows)."""
    try:
        arrays = codec._decode_two_phase([w], True, None, 16, {key})[0][0]
        a = arrays[key]
        if a.ndim == 0 or a.dtype != ref.dtype or a.ndim != ref.ndim or a.shape[1:] != ref.shape[1:]:   # what np.concatenate rejects
            return "ValueError", None
        return None, a
    except Exception as e:  # noqa: BLE001
        return type(e).__name__, None


def _layout_bytes(codec, w, key):
    ck = (N.ConcatKey * 1)()
    kb = key.encode()
    ck[0].key, ck[0].key_len = kb, len(kb)
    N.check(codec._lib.b200tfs_concat_layout(C.c_char_p(w), 1, (C.c_uint64 * 1)(0), (C.c_uint64 * 1)(len(w)), 1, ck, 0))
    return int(ck[0].bytes) if ck[0].status == N.OK else 0


def test_c_mutants_between_valid_records(codec):
    """Every mutant class, the raising ones included, between copies of its valid seed under the seed's first key: the valid
    records' rows are bit-exact at the offsets the plan gave them, each mutant's status is the error class of its own decode,
    and every byte outside the written ranges keeps its 0xEE fill."""
    import decode_mutants as M

    rng = np.random.default_rng(9)
    checked, seeds_used = {}, 0
    for seed, ms in M.corpus():
        if seed.tensor:
            continue
        key = next(iter(codec.parse_predict_responses([seed.wire])[0].outputs))
        try:
            ref = codec._decode_two_phase([seed.wire], True, None, 16, {key})[0][0][key]
        except ValueError:
            continue               # a seed only the tolerant decode accepts (tensor_content, ...): its mutants map to no strict class
        if ref.ndim == 0:
            continue
        seeds_used += 1
        by_kind = {}
        for m in ms:
            by_kind.setdefault(m.kind, []).append(m)
        picked = [m for kind, lst in sorted(by_kind.items()) for m in (lst if len(lst) <= 12 else [lst[int(i)] for i in rng.choice(len(lst), 12, replace=False)])]
        wires, expect = [seed.wire], [(None, ref)]
        for m in picked:
            wires += [m.record, seed.wire]
            expect += [_key_outcome(codec, m.record, key, ref), (None, ref)]
        total = sum(_layout_bytes(codec, w, key) for w in wires)     # what the plan reserves (a varint decode may fail after that)
        lib, ctx, buf, off, ln, ck, kb, arena, dsts = _c_batch(codec, [seed.wire], [key], caps=[total + 4096])
        buf, off, ln = codec._pack_wires(wires)
        arena = codec.device_array(np.frombuffer(bytes(buf), np.uint8))
        N.check(lib.b200tfs_decode_concat(ctx, arena.ptr, len(wires), off, ln, 1, ck))
        outs, st = _results(codec, len(wires), 1)
        got = dsts[0].copy_to_host()
        written = np.zeros(got.size, bool)
        at = 0                             # rows follow each other with no gap: each reserved range starts where the last ended
        for r, (exc, rows) in enumerate(expect):
            o, s = outs[r], outs[r].status
            label = (seed.name, r, picked[(r - 1) // 2].kind if r % 2 else "valid")
            # a place is reserved for OK outputs, for packed-varint outputs whose decode then failed (contents unspecified) and
            # for varint rows left to the unpack route
            if s == N.OK or (o.flags & N.OF_DEVICE_VARINT):
                assert o.dst_off == at, label
                written[o.dst_off: o.dst_off + o.dst_bytes] = True
                at += o.dst_bytes
            if s == N.E_NONCANONICAL:      # left to the unpack route: a record or a layout the device parse does not take
                assert st[r] == N.E_NONCANONICAL or o.flags & N.OF_UNPACKED or o.dtype == 7, label
                checked[s] = checked.get(s, 0) + 1
                continue
            if exc is None:
                assert s == N.OK, (label, s)
                assert o.dst_bytes == rows.nbytes and got[o.dst_off: o.dst_off + rows.nbytes].tobytes() == rows.tobytes(), label
            else:
                assert exc in _EXC_OF.get(s, ()), (label, s, exc)
            checked[s] = checked.get(s, 0) + 1
        assert (got[~written] == 0xEE).all(), seed.name
    assert seeds_used >= 10, seeds_used
    assert checked.get(N.OK) and checked.get(N.E_PARSE) and checked.get(N.E_SHAPE) and checked.get(N.E_KEY), checked
