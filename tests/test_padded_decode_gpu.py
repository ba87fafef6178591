"""Codec.decode_predict_responses_padded and b200tfs_decode_padded: a batch of PredictResponses with ragged trailing dims decoded into
one padded tensor per key on the device, bit for bit against the definition over the per-response decode (numpy's np.full and
slice assignment)."""
import ctypes as C

import numpy as np
import pytest

from golden_util import entry, ld, mspec, tproto, vi
from min_tfs_client import _native as N
from oracle import wire_oracle as O
from test_concat_decode_gpu import DTYPES, _values

pytestmark = pytest.mark.gpu


def _definition(codec, wires, keys, pad_value=0, pad_to=None, strict=False, out_dtypes=None):
    per = [codec.decode_predict_responses([w], strict=strict, out_dtypes=out_dtypes)[0][0] for w in wires]
    res, shapes = {}, {}
    for k in keys:
        parts = [p[k] for p in per]
        rank = parts[0].ndim
        if rank == 0 or any(p.ndim != rank for p in parts) or len({p.dtype for p in parts}) > 1:
            raise ValueError(k)
        tail = tuple(pad_to[k]) if pad_to and k in pad_to else tuple(max(p.shape[d] for p in parts) for d in range(1, rank))
        a = np.full((sum(p.shape[0] for p in parts), *tail), pad_value, parts[0].dtype)
        r0 = 0
        for p in parts:
            a[(slice(r0, r0 + p.shape[0]),) + tuple(slice(0, d) for d in p.shape[1:])] = p
            r0 += p.shape[0]
        res[k] = a
        shapes[k] = np.array([p.shape for p in parts], np.int64)
    return res, shapes


def _host(a):
    return a.copy_to_host() if hasattr(a, "copy_to_host") else np.asarray(a)


def _check(codec, wires, keys=None, device_route=True, **kw):
    before = codec.padded_device_calls
    got, shapes, specs = codec.decode_predict_responses_padded(wires, keys, **kw)
    keys = list(got) if keys is None else keys
    defn = {k: kw[k] for k in ("pad_value", "pad_to", "strict", "out_dtypes") if k in kw}
    want, want_shapes = _definition(codec, wires, keys, **defn)
    for k in keys:
        g = _host(got[k])
        assert g.dtype == want[k].dtype and g.shape == want[k].shape, k
        assert g.tobytes() == want[k].tobytes(), k
        assert np.array_equal(shapes[k], want_shapes[k]) and shapes[k].dtype == np.int64, k
    assert len(specs) == len(wires)
    if device_route:
        assert codec.padded_device_calls == before + 1
    return got


# ---- dtypes and shapes -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: np.dtype(d).name)
@pytest.mark.parametrize("strict", [False, True])
def test_every_dtype_with_ragged_axis_1(codec, dtype, strict):
    if strict and np.dtype(dtype).kind == "c":
        pytest.skip("strict decode rejects complex outputs")
    rng = np.random.default_rng(1)
    shapes = [(3, 5), (0, 2), (1, 9), (12, 0), (1, 1), (7, 4)]
    wires = [O.build_predict_response([("y", _values(rng, dtype, s))]) for s in shapes]
    # strict float16: half_val read as values, which the device does not write: the response-by-response route
    _check(codec, wires, ["y"], device_route=not (strict and np.dtype(dtype) == np.float16), strict=strict, pad_value=1)


@pytest.mark.parametrize("rank", [1, 2, 3, 4, 16])
def test_ranks(codec, rank):
    rng = np.random.default_rng(rank)
    if rank == 16:
        shapes = [(1,) + (1,) * 13 + (2, 3), (2,) + (1,) * 13 + (3, 1)]
    else:
        shapes = [(r,) + tuple(int(x) for x in rng.integers(0, 5, rank - 1)) for r in (2, 1, 3, 0)]
    wires = [O.build_predict_response([("x", rng.standard_normal(s).astype(np.float32))]) for s in shapes]
    _check(codec, wires, pad_value=-1)


def test_rank_3_ragged_in_both_trailing_axes(codec):
    rng = np.random.default_rng(11)
    wires = [O.build_predict_response([("x", rng.standard_normal((1, t, v)).astype(np.float32))]) for t, v in ((5, 3), (2, 7), (6, 6))]
    _check(codec, wires, pad_value=np.float32(-np.inf))


def test_equal_shapes_equal_the_concatenation(codec):
    rng = np.random.default_rng(12)
    wires = [O.build_predict_response([("s", rng.standard_normal((r, 6)).astype(np.float32)),
                                       ("c", rng.integers(0, 1000, (r, 2), dtype=np.int64))]) for r in (4, 0, 3)]
    got = _check(codec, wires)
    cat, _ = codec.decode_predict_responses_concat(wires)
    for k in ("s", "c"):
        assert got[k].tobytes() == cat[k].tobytes() and got[k].shape == cat[k].shape


# ---- pads and casts ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["zero", "minus_one", "minus_inf", "u64_max", "true", "nan_payload"])
def test_pad_values(codec, case):
    rng = np.random.default_rng(13)
    dtype, pad = {"zero": (np.float32, 0), "minus_one": (np.int32, -1), "minus_inf": (np.float64, -np.inf),
                  "u64_max": (np.uint64, np.uint64(2 ** 64 - 1)), "true": (np.bool_, True),
                  "nan_payload": (np.float32, np.array([0x7FC01234], np.uint32).view(np.float32)[0])}[case]
    wires = [O.build_predict_response([("y", _values(rng, dtype, (1, t)))]) for t in (3, 8, 1)]
    got = _check(codec, wires, pad_value=pad)
    if case == "nan_payload":
        assert (got["y"].view(np.uint32)[0, 3:] == 0x7FC01234).all()


@pytest.mark.parametrize("to", [np.float16, "bfloat16"])
def test_narrowing_casts(codec, to):
    from cast_sweep import f32_patterns

    if to == "bfloat16":
        from min_tfs_client.constants import BFLOAT16

        if BFLOAT16 is None:
            pytest.skip("needs ml_dtypes")
        to = BFLOAT16
    vals = f32_patterns().view(np.float32).ravel()
    parts, at = [], 0
    for t in (7, 0, 13, 5) * 40:
        parts.append(vals[at: at + 4 * t].reshape(1, t, 4))
        at += 4 * t
    wires = [O.build_predict_response([("s", p), ("n", np.arange(p.shape[1], dtype=np.int64)[None])]) for p in parts]
    _check(codec, wires, out_dtypes={"s": to}, pad_value=-2.5)


# ---- varint outputs ----------------------------------------------------------------------------------------------
def _varint_values(rng, dtype, t):
    if np.dtype(dtype) == np.bool_:
        return rng.integers(0, 2, t).astype(np.bool_)
    info = np.iinfo(dtype)
    bits = rng.integers(0, 64 if np.dtype(dtype).itemsize == 8 else 32, t)
    v = np.array([(1 << int(b)) - 1 for b in bits], dtype=np.uint64)        # every varint length from 1 to 10 bytes
    return (v.astype(dtype) if info.min == 0 else v.view(np.int64).astype(dtype)) if np.dtype(dtype).itemsize < 8 else v.view(dtype)


@pytest.mark.parametrize("dtype", [np.int64, np.int32, np.bool_], ids=lambda d: np.dtype(d).name)
def test_varint_outputs_of_every_length(codec, dtype):
    rng = np.random.default_rng(14)
    wires = [O.build_predict_response([("ids", _varint_values(rng, dtype, t)[None]), ("f", rng.standard_normal((1, t)).astype(np.float32))])
             for t in (40, 0, 1, 128, 77)]
    _check(codec, wires, pad_value=7 if dtype != np.bool_ else True)


def test_packed_varints_split_over_several_occurrences(codec):
    def rec(vals, cut):
        body = ld(0x52, b"".join(vi(int(v)) for v in vals[:cut])) + ld(0x52, b"".join(vi(int(v)) for v in vals[cut:]))
        return entry("ids", tproto(9, [1, len(vals)], body)) + mspec()
    # occurrences of different lengths (equally long ones at equal distances coalesce into a row of pieces: another route)
    wires = [rec([1, 300, 2 ** 40, -1 & (2 ** 64 - 1), 5], 2), rec([7, 300], 1), rec(list(range(500)), 250)]
    got = _check(codec, wires, pad_value=-3)
    assert got["ids"].shape == (3, 500)


def test_one_long_record_among_short_ones(codec):
    rng = np.random.default_rng(15)
    ts = [3, 65536, 1, 17]
    wires = [O.build_predict_response([("tokens", rng.integers(0, 50000, (1, t), dtype=np.int64))]) for t in ts]
    _check(codec, wires, pad_value=-1)


# ---- batch shape -------------------------------------------------------------------------------------------------
def test_4096_records_two_keys(codec):
    rng = np.random.default_rng(16)
    wires = [O.build_predict_response([("tokens", rng.integers(0, 50000, (1, int(t)), dtype=np.int64)),
                                       ("scores", rng.standard_normal((1, int(t))).astype(np.float32))])
             for t in rng.integers(1, 64, 4096)]
    _check(codec, wires, pad_value=0)


def test_eight_keys_in_shuffled_map_orders(codec):
    rng = np.random.default_rng(17)
    keys = [f"k{i}" for i in range(8)]
    wires = []
    for r in range(6):
        outs = [(k, _values(rng, DTYPES[i % 11], (1 + i % 2, int(rng.integers(0, 6))))) for i, k in enumerate(keys)]
        rng.shuffle(outs)
        wires.append(O.build_predict_response(outs))
    _check(codec, wires, keys, pad_value=1)


# ---- pad_to ------------------------------------------------------------------------------------------------------
def test_pad_to_larger_than_the_batch_maximum_and_a_record_that_exceeds_it(codec):
    rng = np.random.default_rng(18)
    wires = [O.build_predict_response([("l", rng.standard_normal((1, t, 3)).astype(np.float32))]) for t in (4, 9, 2)]
    _check(codec, wires, pad_to={"l": (16, 5)}, pad_value=0.5)
    canary = np.full((3, 8, 3), 1234.5, np.float32)
    before = codec.padded_device_calls
    with pytest.raises(ValueError):
        codec.decode_predict_responses_padded(wires, pad_to={"l": (8, 3)}, out={"l": canary})
    assert (canary == 1234.5).all() and codec.padded_device_calls == before


# ---- destinations ------------------------------------------------------------------------------------------------
def test_device_result_torch_out_and_pinned(codec):
    rng = np.random.default_rng(19)
    wires = [O.build_predict_response([("s", rng.standard_normal((1, t, 10)).astype(np.float32))]) for t in (4, 5, 6)]
    want, _ = _definition(codec, wires, ["s"], pad_value=-1)
    got, _, _ = codec.decode_predict_responses_padded(wires, device=True, pad_value=-1)
    assert hasattr(got["s"], "__cuda_array_interface__")
    assert got["s"].copy_to_host().tobytes() == want["s"].tobytes()
    pinned = codec.pinned_empty((3, 6, 10), np.float32)
    got, _, _ = codec.decode_predict_responses_padded(wires, out={"s": pinned}, pad_value=-1)
    assert got["s"] is pinned and pinned.tobytes() == want["s"].tobytes()
    torch = pytest.importorskip("torch")
    if torch.cuda.is_available():
        t = torch.full((3, 6, 10), 99.0, dtype=torch.float32, device="cuda")
        got, _, _ = codec.decode_predict_responses_padded(wires, out={"s": t}, pad_value=-1)
        torch.cuda.synchronize()
        assert got["s"] is t and t.cpu().numpy().tobytes() == want["s"].tobytes()


# ---- routes ------------------------------------------------------------------------------------------------------
def _same_outcome(codec, wires, keys=None, **kw):
    before = codec.padded_device_calls
    try:
        want = _definition(codec, wires, keys or [], **kw)
        exc = None
    except Exception as e:  # noqa: BLE001
        exc = type(e)
    if exc is not None:
        with pytest.raises(exc):
            codec.decode_predict_responses_padded(wires, keys, **kw)
    else:
        got, shapes, _ = codec.decode_predict_responses_padded(wires, keys, **kw)
        for k in keys:
            assert _host(got[k]).tobytes() == want[0][k].tobytes() and np.array_equal(shapes[k], want[1][k])
    assert codec.padded_device_calls == before


def test_response_by_response_cases(codec):
    f = lambda *s: np.arange(int(np.prod(s)), dtype=np.float32).reshape(s)  # noqa: E731
    good = O.build_predict_response([("a", f(1, 3))])
    nine = O.build_predict_response([(f"k{i}", f(1, i + 1)) for i in range(9)])
    _same_outcome(codec, [nine, O.build_predict_response([(f"k{i}", f(2, 1)) for i in range(9)])], ["k0", "k3"])
    deep = O.build_predict_response([("a", np.ones((1,) * 17 + (2,), np.float32))])
    _same_outcome(codec, [deep, O.build_predict_response([("a", np.ones((2,) + (1,) * 16 + (1,), np.float32))])], ["a"])
    tc = entry("a", O.encode_tensor_proto(f(1, 4), tensor_content=True)) + mspec()
    _same_outcome(codec, [good, tc], ["a"])
    strs = entry("s", tproto(7, [1, 2], ld(0x42, b"ab") + ld(0x42, b"x"))) + mspec()
    _same_outcome(codec, [strs, strs], ["s"])
    unpacked = entry("ids", tproto(9, [1, 3], b"\x50" + vi(5) + b"\x50" + vi(300) + b"\x50" + vi(7))) + mspec()
    _same_outcome(codec, [O.build_predict_response([("ids", np.ones((1, 2), np.int64))]), unpacked], ["ids"])
    _same_outcome(codec, [good, good[:-3]], ["a"])
    _same_outcome(codec, [good, O.build_predict_response([("a", f(1, 3, 1))])], ["a"])
    _same_outcome(codec, [good, O.build_predict_response([("a", np.ones((1, 2), np.float64))])], ["a"])


# ---- C level -----------------------------------------------------------------------------------------------------
def _c_keys(codec, wires, keys, dims, dtype_size, fill=0xEE, extra=512, pad=0x5A):
    lib, ctx = codec._lib, codec.ctx
    buf, off, ln = codec._pack_wires(wires)
    pk = (N.PadKey * len(keys))()
    kb = [k.encode() for k in keys]
    dsts = []
    for i, k in enumerate(kb):
        pk[i].key, pk[i].key_len = k, len(k)
        cap = int(np.prod(dims[i])) * dtype_size[i]
        d = codec.device_array(np.full(cap + extra, fill, np.uint8))
        dsts.append(d)
        pk[i].dst, pk[i].dst_cap, pk[i].rank = d.ptr, cap, len(dims[i])
        for a in range(1, len(dims[i])):
            pk[i].dims[a] = dims[i][a]
        C.memmove(pk[i].pad_bits, bytes([pad]) * 16, 16)
    arena = codec.device_array(np.frombuffer(bytes(buf), np.uint8))
    return lib, ctx, buf, off, ln, pk, kb, arena, dsts


def _results(codec, n, nk):
    outs, specs, st = (N.Output * (n * nk))(), (N.ModelSpec * n)(), (C.c_int32 * n)()
    N.check(codec._lib.b200tfs_padded_results(codec.ctx, n, nk, outs, specs, st))
    return outs, st


def test_c_canary_every_used_byte_written_once_and_nothing_past_them(codec):
    rng = np.random.default_rng(20)
    wires = [O.build_predict_response([("s", rng.standard_normal((1, t, 3)).astype(np.float32)),
                                       ("c", rng.integers(0, 1000, (1, t), dtype=np.int64))]) for t in (5, 0, 9, 2)]
    dims = [(4, 9, 3), (4, 9)]
    lib, ctx, buf, off, ln, pk, kb, arena, dsts = _c_keys(codec, wires, ["s", "c"], dims, [4, 8])
    before = codec.kernel_launches()
    N.check(lib.b200tfs_decode_padded(ctx, arena.ptr, len(wires), off, ln, 2, pk))
    outs, st = _results(codec, len(wires), 2)
    assert codec.kernel_launches() - before == 6
    assert all(outs[j].status == N.OK for j in range(8))
    want, shapes = _definition(codec, wires, ["s", "c"], pad_value=np.float32(np.frombuffer(b"\x5a" * 4, np.float32)[0]))
    want_c, _ = _definition(codec, wires, ["c"], pad_value=np.frombuffer(b"\x5a" * 8, np.int64)[0])
    for i, (k, w) in enumerate((("s", want["s"]), ("c", want_c["c"]))):
        got = dsts[i].copy_to_host()
        assert got[: w.nbytes].tobytes() == w.tobytes(), k      # pads written (the canary is 0xEE, the pad 0x5A)
        assert (got[w.nbytes:] == 0xEE).all(), k
    for r in range(len(wires)):             # each record's own shape
        assert list(outs[r * 2].dims)[:3] == list(shapes["s"][r]) and list(outs[r * 2 + 1].dims)[:2] == list(shapes["c"][r])


def test_c_trailing_dim_above_dims_is_e_size(codec):
    rng = np.random.default_rng(21)
    wires = [O.build_predict_response([("s", rng.standard_normal((1, t)).astype(np.float32))]) for t in (3, 8, 2)]
    lib, ctx, buf, off, ln, pk, kb, arena, dsts = _c_keys(codec, wires, ["s"], [(3, 4)], [4])
    N.check(lib.b200tfs_decode_padded(ctx, arena.ptr, 3, off, ln, 1, pk))
    outs, st = _results(codec, 3, 1)
    assert [outs[r].status for r in range(3)] == [N.OK, N.E_SIZE, N.OK]
    assert outs[2].dst_off == 16
    got = dsts[0].copy_to_host()
    assert (got[32:] == 0xEE).all()


def test_c_graph_replay_adapts_to_new_trailing_dims(codec):
    from min_tfs_client.codec import Codec

    x = np.arange(24, dtype=np.float32)
    a = [O.build_predict_response([("l", x.reshape(1, 6, 4)), ("ids", np.array([[1, 2, 300]], np.int64))]),
         O.build_predict_response([("l", x.reshape(1, 4, 6)), ("ids", np.array([[300, 300, 1]], np.int64))])]
    b = [O.build_predict_response([("l", x.reshape(1, 4, 6)), ("ids", np.array([[70000, 1]], np.int64))]),
         O.build_predict_response([("l", x.reshape(1, 6, 4)), ("ids", np.array([[1, 1, 1, 1, 1]], np.int64))])]
    assert [len(w) for w in a] == [len(w) for w in b]
    gc = Codec(0)           # a captured graph pins the context's scratch buffers: keep it off the shared codec
    dims = [(2, 8, 8), (2, 8)]
    lib, ctx, buf, off, ln, pk, kb, arena, dsts = _c_keys(gc, a, ["l", "ids"], dims, [4, 8], pad=0)
    N.check(lib.b200tfs_decode_padded(ctx, arena.ptr, 2, off, ln, 2, pk))
    _results(gc, 2, 2)
    N.check(lib.b200tfs_capture_begin(ctx))
    N.check(lib.b200tfs_decode_padded(ctx, arena.ptr, 2, off, ln, 2, pk))
    g = C.c_void_p()
    N.check(lib.b200tfs_capture_end(ctx, C.byref(g)))
    buf2, _, _ = gc._pack_wires(b)
    N.check(lib.b200tfs_memcpy_h2d(ctx, arena.ptr, buf2.ctypes.data, buf2.nbytes))
    N.check(lib.b200tfs_graph_launch(ctx, g))
    outs, st = _results(gc, 2, 2)
    N.check(lib.b200tfs_graph_destroy(g))
    assert all(outs[j].status == N.OK for j in range(4))
    assert list(outs[0].dims)[:3] == [1, 4, 6] and list(outs[3].dims)[:2] == [1, 5]
    want, _ = _definition(codec, b, ["l", "ids"], pad_to={"l": (8, 8), "ids": (8,)})
    assert dsts[0].copy_to_host()[: want["l"].nbytes].tobytes() == want["l"].tobytes()
    assert dsts[1].copy_to_host()[: want["ids"].nbytes].tobytes() == want["ids"].tobytes()
    del arena, dsts
    gc.close()


_EXC_OF = {N.E_PARSE: ("DecodeError",), N.E_SHAPE: ("ValueError", "TypeError"), N.E_DTYPE: ("ValueError",), N.E_KEY: ("KeyError",),
           N.E_RANGE: ("OverflowError",)}


def test_c_mutants_statuses_agree_and_nothing_is_stored_outside_the_reported_ranges(codec):
    import decode_mutants as M

    rng = np.random.default_rng(22)
    checked, seeds_used = {}, 0
    for seed, ms in M.corpus():
        if seed.tensor:
            continue
        key = next(iter(codec.parse_predict_responses([seed.wire])[0].outputs))
        try:
            ref = codec._decode_two_phase([seed.wire], True, None, 16, {key})[0][0][key]
        except ValueError:
            continue
        if ref.ndim == 0 or ref.ndim > 4 or ref.dtype.kind in "USO" or ref.size > 4096:
            continue
        seeds_used += 1
        picked = [ms[int(i)] for i in rng.choice(len(ms), min(len(ms), 40), replace=False)]
        wires = [seed.wire]
        for m in picked:
            wires += [m.record, seed.wire]
        tail = tuple(4 * d for d in ref.shape[1:])
        rows = 4 * len(wires)
        dims = (rows,) + tail
        lib, ctx, buf, off, ln, pk, kb, arena, dsts = _c_keys(codec, [seed.wire], [key], [dims], [ref.dtype.itemsize])
        buf, off, ln = codec._pack_wires(wires)
        arena = codec.device_array(np.frombuffer(bytes(buf), np.uint8))
        N.check(lib.b200tfs_decode_padded(ctx, arena.ptr, len(wires), off, ln, 1, pk))
        outs, st = _results(codec, len(wires), 1)
        got = dsts[0].copy_to_host()
        pitch = int(np.prod(tail, dtype=np.int64)) * ref.dtype.itemsize
        used = 0
        for r, w in enumerate(wires):
            o, s = outs[r], outs[r].status
            if s == N.OK or (o.flags & N.OF_DEVICE_VARINT):
                assert o.dst_off == used * pitch, (seed.name, r)
                used += int(o.dims[0])
            if s == N.E_NONCANONICAL or s == N.E_SIZE:
                continue
            try:
                a = codec._decode_two_phase([w], True, None, 16, {key})[0][0][key]
                exc = None if (a.ndim == ref.ndim and a.dtype == ref.dtype) else "ValueError"
            except Exception as e:  # noqa: BLE001
                exc = type(e).__name__
            if exc is None:
                assert s == N.OK, (seed.name, r, s)
                sl = got[o.dst_off: o.dst_off + pitch * a.shape[0]].view(ref.dtype).reshape((a.shape[0],) + tail)
                assert sl[(slice(None),) + tuple(slice(0, d) for d in a.shape[1:])].tobytes() == a.tobytes(), (seed.name, r)
            else:
                assert exc in _EXC_OF.get(s, ()), (seed.name, r, s, exc)
            checked[s] = checked.get(s, 0) + 1
        assert (got[used * pitch:] == 0xEE).all(), seed.name
    assert seeds_used >= 5, seeds_used
    assert checked.get(N.OK) and checked.get(N.E_PARSE), checked
