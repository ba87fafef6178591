"""tf.Example requests (Classify / Regress and Predict) encoded on the GPU at the edges of their four kernels, compared byte for
byte with the numpy reference of example_ref.py.  Every encode runs over an arena filled with a canary byte, with 64 KB of
slack past arena_cap: every byte outside every [rec_off, rec_off + rec_len) must still hold it afterwards.  Each case asks the
geometry model of example_ref.py whether it reached the edge it is named for.

Edges, and the case that reaches each:
  ex_write_example, features per warp pass (32)         test_feature_chunks: 31..200 features, every kind on both sides of a
                                                        chunk boundary, empty payloads there, integer columns in every chunk
  nested lengths at varint widths                       test_nested_lengths_at_varint_widths: P, list, Feature, map entry,
                                                        Features and Example at 127|128, 16383|16384, 2097151|2097152
  feature keys of 2- and 3-byte lengths                 test_long_keys: keys of 127, 128, 16383 and 16384 bytes
  request lengths at varint widths                      test_request_lengths_at_varint_widths: inner and outer at 127|128,
                                                        16383|16384, 2^21 - 1|2^21, 2^28 - 1|2^28 (268 MB float-only
                                                        requests); model names and Predict keys of 127 and 128 bytes
  ex_emit: a batch ending exactly at kExStage           test_emit_image_phases (S = 5459, three examples a span)
  ex_emit: a second batch only for the start phase,     test_emit_image_phases (spans of 16377 bytes at every phase)
           carried partial vectors of 1..15 bytes
  ex_emit: in place only because of the phase           test_emit_image_phases (examples of 16377 bytes)
  ex_emit: examples larger than the image               test_emit_image_phases (16401 bytes, starting and ending at every phase)
  ex_emit: one 16-byte vector stored by 3+ CTAs         test_emit_image_phases (ragged, ex_max > kExStage / 2, 12 and 15 bytes)
  count / scan tiles, frame lane rounds                 test_count_tiles: n around 32 and 1024, 32769 (two lane rounds)
  ex_scan_kernel: a second carry round                  test_two_carry_rounds: 1 049 601 examples behind another request
  carry never crosses requests                          test_tiles_of_several_requests: 1200 tiles in three requests
  count / emit <true> and <false>                       test_both_instantiations
  ex_frame_kernel: device-side E_TOOBIG                 test_message_of_two_gib: 0x7FFFFFFF bytes encoded, 0x80000000 refused
  a captured encode replayed with new lengths           test_graph_replay: spans from one batch to two, examples into and
                                                        out of the in-place path
  the Python entry point                                test_through_the_codec: chunks, emit phases, tiles, shared vectors

Unreachable under today's host planning (the model asserts it, tests/test_example_reference_cpu.py): ex_emit's in-place path
never flushes bytes of earlier examples of its span.  A span of one example (per = 1) has none, and with per >= 2 no example
exceeds kExStage / 2, so none can miss the image after bytes of the same span.
"""
import ctypes as C

import numpy as np
import pytest

import example_ref as R
from devutil import Dev
from min_tfs_client import _native as N
from min_tfs_client.codec import RaggedColumn, _example_columns

pytestmark = pytest.mark.gpu

CANARY = 0xA5
SLACK = 1 << 16
CHUNK = 1 << 28      # bytes compared at a time


@pytest.fixture(scope="module")
def dev():
    d = Dev()
    yield d
    d.close()


def _torch():
    import torch

    return torch


def _on_device(d):
    """the input dict with every array (and ragged lengths) in device memory, as the async entry point reads them"""
    torch = _torch()

    def up(a):
        return torch.from_numpy(np.array(a)).cuda()        # a copy keeps a 0-d array 0-d

    return {k: RaggedColumn(up(v.values), up(v.lengths)) if isinstance(v, RaggedColumn) else up(np.asarray(v)) for k, v in d.items()}


class Item:
    def __init__(self, d, key=None, name="m", version=1, grpc=False, order="deterministic"):
        self.d, self.key, self.name, self.version, self.grpc, self.order = d, key, name, version, grpc, order
        self.plan = R.ReqPlan(name, version, d, key, grpc)


def _call(dev, items, device_dicts=None):
    """the structs of one call (device_dicts: the items' inputs already in device memory), and its arena_cap"""
    n = len(items)
    keep, structs, rg, tg = [], [], [], []
    for i, it in enumerate(items):
        dd = device_dicts[i] if device_dicts else _on_device(it.d)
        m, preps = _example_columns(dd)
        feats = (N.Feature * max(len(preps), 1))(*[p[0] for p in preps])
        nb = it.name.encode()
        structs.append(N.ExampleRequest(model_name=nb, model_name_len=len(nb), has_version=int(it.version is not None),
                                        order=N.ORDER_GIVEN if it.order == "given" else N.ORDER_UPB, version=it.version or 0,
                                        n_examples=m, n_features=len(preps), flags=N.RF_GRPC_FRAME if it.grpc else 0, features=feats))
        rg += [p[3] or N.Ragged() for p in preps]
        kb = None if it.key is None else it.key.encode()
        tg.append(N.ExampleTarget(kind=N.EXAMPLES_PREDICT_STRING, key=kb, key_len=len(kb)) if kb is not None else N.ExampleTarget())
        keep.append((dd, preps, feats, nb, kb))
    reqs, tga = (N.ExampleRequest * n)(*structs), (N.ExampleTarget * n)(*tg)
    rga = (N.Ragged * len(rg))(*rg) if any(g.lengths for g in rg) else None
    cap = C.c_uint64()
    N.check(dev.lib.b200tfs_example_target_arena_size(n, reqs, tga, C.byref(cap)))
    assert cap.value == R.plan([it.plan for it in items])
    return (reqs, rga, tga, keep), cap.value


def _results(dev, items, arena):
    """(status, rec_off, rec_len) of the last encode, after checking that every byte outside the records holds the canary.  A
    refused request (rec_len 0) owns its whole slot: its examples may have been written there before it was refused."""
    n = len(items)
    off, ln = (C.c_uint64 * n)(), (C.c_uint64 * n)()
    st = dev.lib.b200tfs_encode_results(dev.ctx, n, off, ln)
    at = 0
    owned = [(off[i], off[i] + ln[i]) if ln[i] else (it.plan.slot_off, it.plan.slot_end) for i, it in enumerate(items)]
    for a, b in sorted(owned) + [(len(arena), len(arena))]:
        assert a >= at and not bool((arena[at:a] != CANARY).any()), (at, a)
        at = b
    return st, list(off), list(ln)


def _canary_arena(cap):
    torch = _torch()
    arena = torch.full((cap + SLACK,), CANARY, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    return arena


def encode(dev, items):
    """encode items in one call over a canary-filled arena; returns (status, arena, rec_off, rec_len) after the canary check"""
    (reqs, rga, tga, keep), cap = _call(dev, items)
    arena = _canary_arena(cap)
    N.check(dev.lib.b200tfs_encode_example_targets_async(dev.ctx, len(items), reqs, rga, tga, arena.data_ptr(), cap))
    st, off, ln = _results(dev, items, arena)
    return st, arena, off, ln


def same(arena, off, ln, ref_chunks):
    """do arena[off, off + ln) and the concatenated reference chunks hold the same bytes?"""
    at = off
    for c in ref_chunks:
        c = np.asarray(c, np.uint8)
        for a in range(0, len(c), CHUNK):
            part = c[a: a + CHUNK]
            if at + len(part) > off + ln or not np.array_equal(arena[at: at + len(part)].cpu().numpy(), part):
                return False
            at += len(part)
    return at == off + ln


def check(dev, items, done=None):
    """encode items (done: the status, arena and records of an encode already run), compare every request with the reference;
    returns each request's example sizes"""
    st, arena, off, ln = done or encode(dev, items)
    assert st == N.OK, N.last_error()
    sizes = []
    for r, it in enumerate(items):
        S, flat = R.example_bytes(it.d, it.order, 0x0A if it.key is None else 0x42)
        el = int(S.sum())
        pre = R.prefix(it.name, it.version, len(S), el, it.key, it.grpc)
        assert off[r] + ln[r] == it.plan.anchor + el and ln[r] == len(pre) + el, r
        assert same(arena, off[r], ln[r], [np.frombuffer(pre, np.uint8), flat]), r
        sizes.append(S)
    return sizes


def both(d, **kw):
    """the same input as an example_list and as a Predict request"""
    return [Item(d, **kw), Item(d, key="examples", **kw)]


@pytest.mark.parametrize("n_feat", [31, 32, 33, 63, 64, 65, 200])
def test_feature_chunks(dev, n_feat):
    items = []
    for rot in range(len(R.KINDS)):
        d = R.chunk_case(n_feat, rot, seed=n_feat + rot)
        items += both(d, grpc=rot == 1)
    check(dev, items)
    q = items[0].plan
    assert R.chunks(q) == -(-n_feat // 32)
    for c in range(32, n_feat, 32):      # every kind on lane 31 and on lane 0 of every chunk boundary
        assert {R.KINDS[(c - 1 + rot) % 6] for rot in range(6)} == {R.KINDS[(c + rot) % 6] for rot in range(6)} == set(R.KINDS)
    given = dict(reversed(list(R.chunk_case(n_feat, 0, seed=1).items())))
    check(dev, [Item(given, order="given"), Item(given, key="k", order="given")])


@pytest.mark.parametrize("targets", [(127, 128, 16383, 16384), (2_097_151, 2_097_152)], ids=["1-2-3", "3-4"])
def test_nested_lengths_at_varint_widths(dev, targets):
    d, want = R.nested_case(targets)
    items = both(d)
    sizes = check(dev, items)
    n, cols = R.columns(d)
    L = R.nested(cols, n)
    for i, (q, t) in enumerate(want):
        assert (L[q][0, i] if L[q].ndim == 2 else L[q][i]) == t, (q, t)
    if targets[0] > R.K_STAGE:       # the 2 MB examples are written in place
        assert all(len(R.emit(it.plan, S)["in_place"]) == n for it, S in zip(items, sizes))


def test_long_keys(dev):
    rng = np.random.default_rng(3)
    d = {c * L: rng.standard_normal((5, 2)).astype(np.float32) if i % 2 else rng.integers(-9, 1 << 30, (5, 2))
         for i, (c, L) in enumerate(zip("abcd", (127, 128, 16383, 16384)))}
    d["a"] = np.float32(1)          # a prefix of the 127-byte key
    check(dev, both(d) + [Item(d, order="given", grpc=True)])
    assert sorted(set(R.vlen([len(k) for k in d]))) == [1, 2, 3]


@pytest.mark.parametrize("target", [127, 128, 16383, 16384, (1 << 21) - 1, 1 << 21, (1 << 28) - 1, 1 << 28])
def test_request_lengths_at_varint_widths(dev, target):
    items = []
    for q in ("inner", "outer"):
        for key in (None, "e"):
            items.append(Item(R.request_case(q, target, key), key=key))
    for name_len in (127, 128):
        items.append(Item(R.fixed_size(100, 2), name="n" * name_len, version=None))
        items.append(Item(R.fixed_size(100, 2), key="p" * name_len, grpc=True))
    sizes = check(dev, items)
    for it, q, S in zip(items, ("inner", "inner", "outer", "outer"), sizes):
        assert R.request_lengths(it.plan, int(S.sum()), it.key)[q] == target


def test_emit_image_phases(dev):
    # three examples of 5459 bytes a span: spans of 16377 bytes at every phase (9k mod 16), a batch ending exactly at
    # kExStage (phase 7), a second batch only for the phase (phases 8..15), carried partial vectors of 1..15 bytes
    spans = R.fixed_size(5459, 3 * 16 * 2)
    # one example a span: in place only for the phase (16377 bytes), larger than the image at every phase (16401 bytes)
    fit = R.fixed_size(16377, 32, seed=1)
    big = R.fixed_size(16401, 32, seed=2)
    # ragged, ex_max > kExStage / 2, examples of a few bytes: one 16-byte vector stored by several CTAs
    tiny = {"": RaggedColumn(np.ones((64, 1000), np.int64), np.random.default_rng(3).integers(0, 2, 64))}   # 12 or 15 bytes
    items = both(spans) + both(fit) + both(big) + both(tiny) + [Item(spans, grpc=True, version=None)]
    sizes = check(dev, items)
    m = [R.emit(it.plan, S) for it, S in zip(items, sizes)]
    for k in (0, 1):
        assert items[k].plan.per == 3 and m[k]["span_phases"] == set(range(16))
        assert m[k]["full"] and m[k]["multi"] and m[k]["carried"] >= set(range(1, 16)), m[k]["carried"]
        assert not m[k]["in_place"]
        assert m[2 + k]["in_place"] and m[2 + k]["batches"] and len(m[2 + k]["in_place"]) < 32     # the phase decides
        assert {s for s, _, _ in m[4 + k]["in_place"]} == {e for _, e, _ in m[4 + k]["in_place"]} == set(range(16))
        assert items[6 + k].plan.per == 1 and m[6 + k]["sharers"] >= 3
    assert all(R.covers_once(it.plan, S, mm["stores"]) for it, S, mm in zip(items, sizes, m))


@pytest.mark.parametrize("n", [1, 31, 32, 33, 1023, 1024, 1025, 2047, 2049, 32769])
def test_count_tiles(dev, n):
    d = R.counted_case(n, seed=n)
    items = both(d) + [Item(R.counted_case(n % 97 + 1, seed=1), grpc=True)]
    check(dev, items)
    q = items[0].plan
    assert q.counted and q.n_tiles == -(-n // R.K_TILE)
    assert R.frame_rounds(q) == (2 if n == 32769 else 1)


def test_two_carry_rounds(dev):
    n = R.K_TILE * (R.K_TILE + 1) + 1
    items = [Item(R.counted_case(5000, seed=1)), Item(R.counted_case(n, seed=2), key="examples")]
    check(dev, items)
    R.plan([it.plan for it in items])
    q = items[1].plan
    # its carry rounds start at absolute tile 5, off the kExTile grid, and its tiles cross absolute tile 1024
    assert q.first_tile == 5 and max(R.scan_rounds(q)) == 2 and q.first_tile + q.n_tiles > R.K_TILE


def test_tiles_of_several_requests(dev):
    items = [Item(R.counted_case(400 * R.K_TILE, seed=s), key="x" if s == 1 else None) for s in range(3)]
    check(dev, items)
    assert sum(it.plan.n_tiles for it in items) > R.K_TILE and all(max(R.scan_rounds(it.plan)) == 1 for it in items)


def test_both_instantiations(dev):
    rng = np.random.default_rng(7)
    dense = {"i": rng.integers(-(1 << 50), 1 << 50, (3000, 3)), "x": rng.standard_normal((3000, 2)).astype(np.float32)}
    flt = R.fixed_size(5459, 100)
    rag = {"r": RaggedColumn(rng.integers(0, 1 << 20, (2000, 9)), rng.integers(0, 10, 2000)), "h": rng.standard_normal(2000).astype(np.float16)}
    items = both(dense) + both(flt)
    alone = [check(dev, [it]) for it in items]
    without = check(dev, items)                          # <false>: no ragged column in the call
    with_r = check(dev, items + both(rag))              # <true>
    assert [a[0].tolist() for a in alone] == [s.tolist() for s in without] == [s.tolist() for s in with_r[:4]]


def test_message_of_two_gib(dev):
    """A counted request that passes the host's check (examples at their shortest fit 2 GiB) and whose real message is
    0x7FFFFFFF bytes is encoded; one byte more is E_TOOBIG on the device, and a good request beside it is unaffected."""
    R_ELEMS = 100
    one = {"a": np.full((1, R_ELEMS), -1, np.int8), "b": np.full((1, 1), 127, np.int16)}
    S = int(R.example_bytes(one)[0][0])        # with b = 128: S + 1
    spec = R.model_spec("m", 1)
    for msg, want in ((R.PROTO_LIMIT, N.OK), (R.PROTO_LIMIT + 1, N.E_TOOBIG)):
        el = msg - len(spec) - 12                     # 12 = two tags and two 5-byte lengths
        n = el // S
        m = el - n * S                                # examples with a 2-byte int16 varint
        assert 0 < m < n
        d = {"a": np.full((n, R_ELEMS), -1, np.int8), "b": np.where(np.arange(n) < m, 128, 127).astype(np.int16)[:, None]}
        good = R.counted_case(300, seed=3)
        items = [Item(d), Item(good, key="g")]
        q = items[0].plan
        assert n * q.ex_min <= R.PROTO_LIMIT
        assert R.request_lengths(q, el)["msg"] == msg
        st, arena, off, ln = encode(dev, items)
        assert st == want, N.last_error()
        ref = R.request_bytes("m", 1, good, key="g")
        assert arena[off[1]: off[1] + ln[1]].cpu().numpy().tobytes() == ref
        if want == N.E_TOOBIG:
            assert off[0] == ln[0] == 0
            continue
        ex = [R.example_bytes({k: v[i: i + 1] for k, v in d.items()})[1] for i in (0, n - 1)]    # b = 128, b = 127
        pattern = (np.arange(n) >= m).astype(np.int64)
        chunks = [np.frombuffer(R.prefix("m", 1, n, el), np.uint8)]
        chunks += (R.examples_chunk(ex, pattern, i, min(i + (1 << 18), n)) for i in range(0, n, 1 << 18))
        assert ln[0] == msg and same(arena, off[0], ln[0], chunks)
        del arena


def test_graph_replay(dev):
    """One captured encode replayed with new values and lengths: the spans of request a (three examples each) go from one batch
    to two, the examples of request b (one a span, larger than the image at their longest) into and out of the in-place path."""
    torch = _torch()
    rng = np.random.default_rng(23)
    n, Ma, Mb = 60, 1360, 4096
    bufs = [torch.zeros((n, Ma), dtype=torch.float32, device="cuda"), torch.zeros(n, dtype=torch.int64, device="cuda"),
            torch.zeros((n, Mb), dtype=torch.float32, device="cuda"), torch.zeros(n, dtype=torch.int64, device="cuda")]
    dev_dicts = [{"a": RaggedColumn(bufs[0], bufs[1])}, {"b": RaggedColumn(bufs[2], bufs[3])}]

    def items_of(host):
        return [Item({"a": RaggedColumn(host[0], host[1])}, key="examples"), Item({"b": RaggedColumn(host[2], host[3])}, grpc=True)]

    shapes = [np.zeros((n, Ma), np.float32), np.zeros(n, np.int64), np.zeros((n, Mb), np.float32), np.zeros(n, np.int64)]
    (reqs, rga, tga, keep), cap = _call(dev, items_of(shapes), dev_dicts)
    arena = _canary_arena(cap)
    N.check(dev.lib.b200tfs_encode_example_targets_async(dev.ctx, 2, reqs, rga, tga, arena.data_ptr(), cap))   # sizes every buffer
    N.check(dev.lib.b200tfs_encode_results(dev.ctx, 2, None, None))
    N.check(dev.lib.b200tfs_capture_begin(dev.ctx))
    N.check(dev.lib.b200tfs_encode_example_targets_async(dev.ctx, 2, reqs, rga, tga, arena.data_ptr(), cap))
    g = C.c_void_p()
    N.check(dev.lib.b200tfs_capture_end(dev.ctx, C.byref(g)))
    seen = {"one batch": False, "two batches": False, "in place": False, "batched": False}
    try:
        for lo_a, lo_b in ((0, 0), (Ma, Mb), (Ma - 8, Mb - 20), (0, 0)):
            host = [rng.standard_normal((n, Ma)).astype(np.float32), rng.integers(lo_a, Ma + 1, n),
                    rng.standard_normal((n, Mb)).astype(np.float32), rng.integers(lo_b, Mb + 1, n)]
            for buf, h in zip(bufs, host):
                buf.copy_(torch.from_numpy(h))
            arena.fill_(CANARY)
            torch.cuda.synchronize()
            N.check(dev.lib.b200tfs_graph_launch(dev.ctx, g))
            items = items_of(host)
            R.plan([it.plan for it in items])
            st, off, ln = _results(dev, items, arena)
            sa, sb = check(dev, items, (st, arena, off, ln))
            ma, mb = R.emit(items[0].plan, sa), R.emit(items[1].plan, sb)
            seen["one batch"] |= ma["multi"] == 0
            seen["two batches"] |= ma["multi"] > 0
            seen["in place"] |= bool(mb["in_place"])
            seen["batched"] |= bool(mb["batches"])
        assert items[0].plan.per == 3 and items[1].plan.per == 1 and all(seen.values()), seen
    finally:
        N.check(dev.lib.b200tfs_graph_destroy(g))


def test_through_the_codec(codec):
    """the Python entry point (host columns staged on the device, the wire copied back) over a subset of the edges"""
    cases = [R.chunk_case(65, 3, seed=4), R.fixed_size(5459, 48), R.fixed_size(16401, 17), R.counted_case(2049, seed=5),
             {"": RaggedColumn(np.ones((64, 1000), np.int64), np.random.default_rng(3).integers(0, 2, 64))}]
    items = [("m", 1, d) for d in cases]
    assert codec.encode_example_requests(items) == [R.request_bytes("m", 1, d) for d in cases]
    got = codec.encode_example_requests(items, predict_input="examples", grpc_frame=True)
    assert got == [R.request_bytes("m", 1, d, key="examples", grpc=True) for d in cases]
    assert codec.encode_example_requests(items[:1], order="given") == [R.request_bytes("m", 1, cases[0], order="given")]
