"""Packed-varint encode and decode on the device at every tile, group and window edge, compared with the numpy reference
(tests/varint_ref.py, pinned to the protobuf runtime by tests/test_varint_reference_cpu.py) byte for byte and value for value.

Encode tiles are 2048 elements and their counters are summed in groups of 256 tiles (524 288 elements); decode tiles are aligned
8 KB windows of the wire, summed in groups of 256 (2 MiB).  Every case asserts that it reaches the edge it is named for.
Decode wires are built by the reference, never by the device encoder, and every decode route is compared with the reference
values, not with another route.
"""
import ctypes as C

import numpy as np
import pytest
from google.protobuf.message import DecodeError

import decode_mutants as D
import varint_ref as V
from devutil import Dev, tensor_struct
from min_tfs_client import _native as N
from min_tfs_client.codec import Codec
from oracle import wire_oracle
from test_device_api_gpu import _encode_requests_device
from test_varint_decode_gpu import K, Single, place, two_phase

pytestmark = pytest.mark.gpu

NP = {3: np.int32, 4: np.uint8, 5: np.int16, 6: np.int8, 17: np.uint16, 9: np.int64, 22: np.uint32, 23: np.uint64, 10: np.bool_,
      19: np.float16}


@pytest.fixture(scope="module")
def dev():
    d = Dev()
    yield d
    d.close()


def launches(dev, ctx=None):
    v = C.c_uint64()
    N.check(dev.lib.b200tfs_kernel_launches(ctx or dev.ctx, C.byref(v)))
    return v.value


def free(dev, p):
    dev.lib.b200tfs_free(dev.ctx, C.c_void_p(p))
    dev.allocs.remove(p)


def mixed(dtype, n, rng):
    """n values of `dtype` whose varints take every length the dtype can have, in random order."""
    t = NP[dtype]
    if dtype == 10:
        return rng.integers(0, 2, n).astype(np.bool_)
    if dtype == 19:
        return rng.integers(0, 1 << 16, n, dtype=np.uint64).astype(np.uint16).view(np.float16)
    info = np.iinfo(t)
    bits = info.bits - (1 if info.min < 0 else 0)
    raw = rng.integers(0, 1 << bits, n, dtype=np.uint64) >> rng.integers(0, bits, n).astype(np.uint64)
    v = raw.astype(t)
    if info.min < 0:
        v = np.where(rng.random(n) < 0.2, -v - 1, v).astype(t)
    return v


# ---- encode -------------------------------------------------------------------------------------------------------------
def encode_protos(dev, arrays, ptrs=None, measure=True):
    """Encode `arrays` (already on the device at `ptrs`, else uploaded) as bare TensorProtos: (wires, packed_len per tensor,
    kernels of the encode that used the measure's counters, kernels of a second encode of the same tensors)."""
    own = ptrs is None
    ptrs = [dev.upload(a) for a in arrays] if own else ptrs
    keep = [tensor_struct(p, a) for p, a in zip(ptrs, arrays)]
    arr = (N.Tensor * len(keep))(*[t for t, _ in keep])
    if measure:
        N.check(dev.lib.b200tfs_measure(dev.ctx, len(keep), arr))
    need = C.c_uint64()
    N.check(dev.lib.b200tfs_tensor_arena_size(len(keep), arr, C.byref(need)))
    arena = dev.malloc(need.value)
    off, ln = (C.c_uint64 * len(keep))(), (C.c_uint64 * len(keep))()
    used = []
    wires = None
    for _ in range(2):
        before = launches(dev)
        N.check(dev.lib.b200tfs_encode_tensor_protos(dev.ctx, len(keep), arr, arena, need.value, off, ln))
        used.append(launches(dev) - before)
        raw = dev.download(arena, need.value)
        got = [bytes(raw[off[i]: off[i] + ln[i]]) for i in range(len(keep))]
        assert wires is None or got == wires          # the encode that counted again writes the same bytes
        wires = got
    free(dev, arena)
    if own:
        for p in ptrs:
            free(dev, p)
    return wires, [arr[i].packed_len for i in range(len(keep))], used[0], used[1]


COUNTS = [1, 31, 32, 33, 2047, 2048, 2049, 4096, 4097, 524287, 524288, 524289, 2 * 524288 + 2049]


@pytest.mark.parametrize("dtype", [9, 3, 22, 23, 5, 6, 4, 17, 10, 19], ids=lambda d: V.NAMES[d])
def test_encode_element_counts_across_tiles_and_groups(dev, dtype):
    rng = np.random.default_rng(dtype)
    counts = COUNTS if dtype in (9, 3) else [1, 31, 32, 33, 2047, 2048, 2049, 524289]
    crossed = 0
    for n in counts:
        a = mixed(dtype, n, rng)
        wires, plen, measured, again = encode_protos(dev, [a])
        assert wires[0] == V.tensor_proto(a, dtype), (dtype, n)
        if dtype != 10:                                     # bool_val takes one byte per element: nothing to measure
            assert plen[0] == V.packed_len(a, dtype), (dtype, n)
            assert again == measured + 1, (dtype, n)       # the measured encode skipped the counting kernel
        crossed += -(-n // V.ENC_TILE) > V.GROUP_TILES
    assert crossed >= 1                                     # the group sums of prefix_share were read


def layout_cases(rng):
    """int64 arrays of whole tiles that aim at the emit kernel's branches: (name, array)."""
    T = V.ENC_TILE
    narrow = rng.integers(0, 1 << 28, 3 * T, dtype=np.int64)
    cases = [("narrow", narrow)]
    # one 5..10-byte value in an otherwise narrow tile: at lane 0, at lane 31 (thread 31 owns elements 248..255), and as
    # element 7 of a thread (blocked layout: thread r owns elements 8r..8r+7)
    wide = {5: 1 << 28, 6: 1 << 35, 7: 1 << 42, 8: 1 << 49, 9: 1 << 56, 10: -1}
    one = rng.integers(0, 1 << 28, 18 * T, dtype=np.int64)
    t = 0
    for L, v in wide.items():
        for at in (0, 8 * 31 + 3, 8 * 77 + 7):
            one[t * T + at] = v
            assert V.varint_lengths(np.array([v]).view(np.uint64))[0] == L
            t += 1
    cases.append(("one_wide", one))
    # values of 2^32 and more in one lane only (the any_hi branch of the 128-bit load path)
    hi = rng.integers(0, 1 << 28, 2 * T, dtype=np.int64)
    hi[8 * 40: 8 * 41] = rng.integers(1 << 32, 1 << 62, 8, dtype=np.int64)
    cases.append(("one_lane_hi", hi))
    # thread r: seven 1-byte values and one of 1 + r % 4 bytes, so thread starts in the shared image take every offset mod 4
    runs = rng.integers(0, 128, 3 * T, dtype=np.int64).reshape(-1, 8)
    r = np.arange(runs.shape[0]) % V.GROUP_TILES
    runs[np.arange(runs.shape[0]), r % 8] = (1 << (7 * (r % 4))) + rng.integers(0, 64, runs.shape[0])
    runs = runs.reshape(-1)
    starts = np.cumsum(V.varint_lengths(runs.view(np.uint64)).reshape(-1, 8).sum(1)) % 4
    assert set(starts.tolist()) == {0, 1, 2, 3}
    cases.append(("offsets_mod4", runs))
    return cases


def test_encode_value_layouts_at_both_source_alignments(dev):
    """The same int64 values from a 16-byte aligned source (128-bit loads) and from an 8-mod-16 one (striped loads and the
    shared-memory transpose): identical bytes, equal to the reference."""
    rng = np.random.default_rng(11)
    for name, a in layout_cases(rng):
        want = V.tensor_proto(a, 9)
        buf = np.zeros(a.size + 2, dtype=np.int64)
        buf[1: 1 + a.size] = a
        p = dev.upload(buf)
        assert p % 16 == 0
        for at in (p + 8, p + 16):
            if at == p + 16:
                N.check(dev.lib.b200tfs_memcpy_h2d(dev.ctx, p + 16, a.ctypes.data, a.nbytes))
                dev.sync()
            wires, plen, _, _ = encode_protos(dev, [a], [at])
            assert wires[0] == want and plen[0] == V.packed_len(a, 9), (name, at - p)
        free(dev, p)


def test_encode_source_offsets_and_misaligned_sources(dev):
    rng = np.random.default_rng(12)
    n = 2 * V.ENC_TILE + 5
    for dtype in (3, 5, 6, 17, 4, 22):
        a = mixed(dtype, n, rng)
        size = a.itemsize
        want = V.tensor_proto(a, dtype)
        raw = np.zeros(a.nbytes + 32, dtype=np.uint8)
        p = dev.upload(raw)
        for shift in range(0, 16, size):
            N.check(dev.lib.b200tfs_memcpy_h2d(dev.ctx, p + shift, a.ctypes.data, a.nbytes))
            dev.sync()
            wires, _, _, _ = encode_protos(dev, [a], [p + shift])
            assert wires[0] == want, (dtype, shift)
        if size > 1:                      # a source not aligned to its element size is refused
            t, dims = tensor_struct(p + 1, a)
            arr = (N.Tensor * 1)(t)
            rc = dev.lib.b200tfs_measure(dev.ctx, 1, arr)
            if rc == N.OK:
                need = C.c_uint64()
                N.check(dev.lib.b200tfs_tensor_arena_size(1, arr, C.byref(need)))
                arena = dev.malloc(need.value)
                off, ln = (C.c_uint64 * 1)(), (C.c_uint64 * 1)()
                rc = dev.lib.b200tfs_encode_tensor_protos(dev.ctx, 1, arr, arena, need.value, off, ln)
                free(dev, arena)
            assert rc == N.E_ARG, (dtype, rc)
        free(dev, p)


def test_encode_forty_jobs_in_one_launch(dev):
    """Jobs of mixed sizes and dtypes, empty ones among them: the tile -> segment table instead of the single job."""
    rng = np.random.default_rng(13)
    sizes = [0, 1, 31, 32, 33, 0, 2047, 2048, 2049, 4097, 5, 0, 70000, 3, 600000] * 3
    dts = [9, 3, 22, 23, 5, 6, 4, 17, 10, 19]
    arrays = [mixed(dts[i % len(dts)], n, rng) for i, n in enumerate(sizes[:40])]
    wires, plen, measured, again = encode_protos(dev, arrays)
    for i, a in enumerate(arrays):
        dt = [9, 3, 22, 23, 5, 6, 4, 17, 10, 19][i % len(dts)]
        assert wires[i] == V.tensor_proto(a, dt) and (dt == 10 or plen[i] == V.packed_len(a, dt)), i
    assert again == measured + 1


def test_encode_never_writes_past_the_measured_length(dev):
    """Measure, rewrite the buffer with longer varints, encode into a canary-filled arena: every framing byte is the reference
    framing for the MEASURED length and no arena byte outside the record changes (the payload bytes are unspecified)."""
    rng = np.random.default_rng(14)
    for n in (2049, 600000):
        a = rng.integers(0, 128, n, dtype=np.int64)
        p = dev.upload(a)
        t, dims = tensor_struct(p, a)
        arr = (N.Tensor * 1)(t)
        N.check(dev.lib.b200tfs_measure(dev.ctx, 1, arr))
        L = arr[0].packed_len
        assert L == n
        b = rng.integers(1 << 40, 1 << 62, n, dtype=np.int64)
        N.check(dev.lib.b200tfs_memcpy_h2d(dev.ctx, p, b.ctypes.data, b.nbytes))
        dev.sync()
        need = C.c_uint64()
        N.check(dev.lib.b200tfs_tensor_arena_size(1, arr, C.byref(need)))
        cap = need.value + 4096
        arena = dev.malloc(cap)
        N.check(dev.lib.b200tfs_memset(dev.ctx, arena, 0xA5, cap))
        off, ln = (C.c_uint64 * 1)(), (C.c_uint64 * 1)()
        N.check(dev.lib.b200tfs_encode_tensor_protos(dev.ctx, 1, arr, arena, need.value, off, ln))
        raw = dev.download(arena, cap)
        head = V.tensor_header(9, [n], L)
        assert ln[0] == len(head) + L
        assert raw[off[0]: off[0] + len(head)].tobytes() == head
        outside = np.ones(cap, dtype=bool)
        outside[off[0]: off[0] + ln[0]] = False
        assert (raw[outside] == 0xA5).all(), n
        free(dev, arena)
        free(dev, p)


def test_encode_requests_at_every_destination_phase(dev):
    """Key lengths 0..15 put the packed payload at every 16-byte phase of the arena; next to a larger float input the varint
    payload is not the record's 128-byte aligned one."""
    rng = np.random.default_rng(15)
    ids = mixed(9, 3 * V.ENC_TILE + 17, rng)
    img = rng.standard_normal(20000).astype(np.float32)
    batch = []
    for k in range(16):
        batch.append(("default", 1, [("k" * k, ids)]))
        batch.append(("default", 1, [("k" * k, ids), ("image", img)]))
    wires, (arena, off, ln) = _encode_requests_device(dev, batch)
    phases = set()
    for i, (_, _, inputs) in enumerate(batch):
        assert wires[i] == wire_oracle.encode_predict_request("default", 1, inputs), i
        phases.add((arena + off[i] + wires[i].index(V.encode(ids, 9)[:64])) % 16)
    assert phases == set(range(16))


def _requests(dev, batch, host=False):
    """N.Request structs for [(model, version, [(key, ndarray)])]; device copies unless `host`."""
    keep, reqs = [], []
    for model, version, inputs in batch:
        ts = []
        for k, a in inputs:
            a = np.ascontiguousarray(a)
            keep.append(a)
            t, dims = tensor_struct(a.ctypes.data if host else dev.upload(a), a, key=k.encode())
            if host:
                t.flags = 0
            keep.append(dims)
            ts.append(t)
        arr = (N.Tensor * max(len(ts), 1))(*ts)
        keep.append(arr)
        name = model.encode()
        keep.append(name)
        reqs.append(N.Request(model_name=name, model_name_len=len(name), has_version=int(version is not None), order=N.ORDER_UPB,
                              version=version or 0, n_inputs=len(ts), flags=0, inputs=arr))
    return (N.Request * len(reqs))(*reqs), keep


def _encode_async(dev, rq, n):
    need = C.c_uint64()
    N.check(dev.lib.b200tfs_request_arena_size(n, rq, C.byref(need)))
    arena = dev.malloc(need.value)
    N.check(dev.lib.b200tfs_encode_requests_async(dev.ctx, n, rq, arena, need.value))
    return arena, need.value


def _results(dev, arena, cap, n):
    off, ln = (C.c_uint64 * n)(), (C.c_uint64 * n)()
    N.check(dev.lib.b200tfs_encode_results(dev.ctx, n, off, ln))
    raw = dev.download(arena, cap)
    return [raw[off[i]: off[i] + ln[i]].tobytes() for i in range(n)]


def test_deferred_encode_across_the_tiny_limit_and_a_large_request(dev):
    rng = np.random.default_rng(16)
    batch = [("m", 3, [("ids", mixed(9, n, rng))]) for n in (V.TINY - 1, V.TINY, V.TINY + 1, V.ENC_TILE + 1)]
    batch.append(("m", None, [("a", mixed(3, V.TINY, rng)), ("b", mixed(6, V.TINY + 1, rng)), ("c", mixed(22, 1, rng))]))
    # a large request: a model name over 1 KB and 72 inputs, most of them tiny packed varints, in one record of the batch
    many = [("t%02d" % i, mixed(9, V.TINY // 8 + 1, rng)) for i in range(64)]
    many += [("u%02d" % i, mixed(3, V.TINY + i, rng)) for i in range(8)]
    batch.append(("model_" + "n" * 1124, 7, many))
    assert sum(a.size for _, a in many if a.size <= V.TINY) > 32 and len(many) > 32
    rq, keep = _requests(dev, batch)
    arena, cap = _encode_async(dev, rq, len(batch))
    got = _results(dev, arena, cap, len(batch))
    for i, (model, version, inputs) in enumerate(batch):
        assert got[i] == wire_oracle.encode_predict_request(model, version, inputs), i
    free(dev, arena)


def test_deferred_encode_graph_replay_changes_lengths_across_a_group():
    dev = Dev()                           # a captured graph pins its context's scratch buffers: a context of its own
    try:
        _graph_replay(dev)
    finally:
        dev.close()


def _graph_replay(dev):
    rng = np.random.default_rng(17)
    n = V.ENC_GROUP_ELEMS + 3 * V.ENC_TILE + 1
    first = rng.integers(0, 128, n, dtype=np.int64)
    batch = [("m", 1, [("ids", first), ("x", np.arange(7, dtype=np.int32))])]
    rq, keep = _requests(dev, batch)
    arena, cap = _encode_async(dev, rq, 1)
    assert _results(dev, arena, cap, 1)[0] == wire_oracle.encode_predict_request("m", 1, batch[0][2])
    N.check(dev.lib.b200tfs_capture_begin(dev.ctx))
    N.check(dev.lib.b200tfs_encode_requests_async(dev.ctx, 1, rq, arena, cap))
    g = C.c_void_p()
    N.check(dev.lib.b200tfs_capture_end(dev.ctx, C.byref(g)))
    try:
        # new values: one byte in the first group, up to ten bytes past it - every later tile moves
        second = first.copy()
        second[V.ENC_GROUP_ELEMS:] = mixed(9, n - V.ENC_GROUP_ELEMS, rng)
        ptr = rq[0].inputs[0].data
        N.check(dev.lib.b200tfs_memcpy_h2d(dev.ctx, ptr, second.ctypes.data, second.nbytes))
        N.check(dev.lib.b200tfs_graph_launch(dev.ctx, g))
        assert _results(dev, arena, cap, 1)[0] == wire_oracle.encode_predict_request("m", 1, [("ids", second), batch[0][2][1]])
    finally:
        N.check(dev.lib.b200tfs_graph_destroy(g))
    free(dev, arena)


def test_host_encode_at_the_host_measure_limit(dev):
    rng = np.random.default_rng(18)
    for n in (V.HOST_MEASURE, V.HOST_MEASURE + 1):
        batch = [("m", 1, [("ids", mixed(9, n, rng)), ("s", mixed(3, 40, rng))])]
        rq, keep = _requests(dev, batch, host=True)
        need = C.c_uint64()
        N.check(dev.lib.b200tfs_request_arena_size(1, rq, C.byref(need)))
        hp = C.c_void_p()
        N.check(dev.lib.b200tfs_host_alloc(need.value, C.byref(hp)))
        try:
            off, ln = (C.c_uint64 * 1)(), (C.c_uint64 * 1)()
            N.check(dev.lib.b200tfs_encode_requests_host_async(dev.ctx, 1, rq, hp, need.value, off, ln))
            dev.sync()
            host = (C.c_uint8 * need.value).from_address(hp.value)
            assert bytes(host[off[0]: off[0] + ln[0]]) == wire_oracle.encode_predict_request("m", 1, batch[0][2]), n
        finally:
            dev.lib.b200tfs_host_free(hp)


# ---- decode -------------------------------------------------------------------------------------------------------------
def record(key, dtype, n, chunks):
    return D.entry(key, D.tproto(dtype, [n], V.field(dtype, chunks))) + D.mspec()


def chunk_offsets(rec, dtype, chunks):
    """Offsets inside `rec` of the value chunks (tag and length prefix skipped)."""
    at, out = 0, []
    for c in chunks:
        head = D.vi((V.DTYPES[dtype][0] << 3) | 2) + D.vi(len(c))
        at = rec.index(head + c, at) + len(head)
        out.append(at)
        at += len(c)
    return out


def windows(addr, length):
    """Decode tiles of a chunk at absolute address `addr`: aligned 8 KB windows from addr & ~15."""
    return (addr % 16 + length + V.DEC_TILE - 1) // V.DEC_TILE


def decode_all_routes(dev, recs, expect, graph=False):
    """Decode `recs` (one varint output "v" each, plus nothing else) by the two-phase route and the single-launch decode with
    the varint switch on (eagerly, and as a graph replay when `graph`); every value equals expect[r] (a numpy array).  Returns
    the absolute address of every record in the arena the routes read."""
    want = [np.ascontiguousarray(e).tobytes() for e in expect]
    got, st, _ = two_phase(dev, recs)
    for r in range(len(recs)):
        assert st[r] == N.OK and got[(r, 0)] == (N.OK, want[r]), ("two-phase", r)
    s = Single(dev, recs)
    try:
        for _ in range(2):
            outs, n_outs, rs, slots = s.run()
            for r in range(len(recs)):
                o = outs[r * K]
                assert rs[r] == N.OK and o.status == N.OK and o.flags & N.OF_DEVICE_VARINT, ("single", r, o.status)
                a = r * s.stride + int(o.dst_off)
                assert slots[a: a + len(want[r])].tobytes() == want[r], ("single", r)
        if graph:
            N.check(dev.lib.b200tfs_sync(s.ctx))
            N.check(dev.lib.b200tfs_capture_begin(s.ctx))
            N.check(dev.lib.b200tfs_decode_responses(s.ctx, s.arena_dev, len(recs), s.off, s.ln, s.dst, s.stride))
            g = C.c_void_p()
            N.check(dev.lib.b200tfs_capture_end(s.ctx, C.byref(g)))
            s.fill()
            N.check(dev.lib.b200tfs_graph_launch(s.ctx, g))
            outs, n_outs, rs, slots = s.results(s.download())
            N.check(dev.lib.b200tfs_graph_destroy(g))
            for r in range(len(recs)):
                o = outs[r * K]
                a = r * s.stride + int(o.dst_off)
                assert o.status == N.OK and slots[a: a + len(want[r])].tobytes() == want[r], ("graph", r)
        return [s.arena_dev + int(s.off[r]) for r in range(len(recs))]
    finally:
        s.close()


def phase_records(dtype, vals, chunks_of, n_phases=16):
    """One record per 16-byte phase of its first chunk's start in the arena place() builds: key lengths are chosen so that
    record i (placed at (7 i) mod 64 past a 256-byte boundary) starts its first chunk at phase i."""
    recs = []
    chunks = chunks_of(vals)
    for i in range(n_phases):
        for k in range(1, 80):
            rec = record("v" * k, dtype, vals.size, chunks)
            if ((7 * i) % 64 + chunk_offsets(rec, dtype, chunks)[0]) % 16 == i % 16:
                recs.append(rec)
                break
        else:
            raise AssertionError(i)
    return recs


def test_decode_chunks_past_a_group_at_every_phase(dev):
    rng = np.random.default_rng(21)
    full = rng.integers(-2 ** 63, 2 ** 63 - 1, 300000, dtype=np.int64, endpoint=True)   # 2.8 MB: past one group of windows
    recs = phase_records(9, full, lambda v: [V.encode(v, 9)])
    addrs = decode_all_routes(dev, recs, [full] * len(recs))
    wire = V.encode(full, 9)
    assert {(a + chunk_offsets(r, 9, [wire])[0]) % 16 for a, r in zip(addrs, recs)} == set(range(16))
    assert windows(addrs[0], len(wire)) > V.GROUP_TILES
    small = rng.integers(0, 128, 2200000).astype(np.int32)     # 2.2 M one-byte values
    recs = phase_records(3, small, lambda v: [V.encode(v, 3)], n_phases=4)
    decode_all_routes(dev, recs, [small] * len(recs), graph=True)


def test_decode_split_fields_with_a_group_edge_in_a_later_chunk(dev):
    rng = np.random.default_rng(22)
    vals = mixed(9, 400000, rng)
    recs, expect = [], []
    for parts in range(2, 9):
        cut = np.linspace(0, vals.size, parts + 1).astype(int)
        chunks = [V.encode(vals[cut[i]: cut[i + 1]], 9) for i in range(parts)]
        rec = record("v", 9, vals.size, chunks)
        recs.append(rec)
        expect.append(vals)
        assert sum(windows(0, len(c)) for c in chunks[:-1]) < V.GROUP_TILES < sum(windows(0, len(c)) for c in chunks)
    decode_all_routes(dev, recs, expect)
    # the concatenated and padded batch decodes, on the device route (never the per-record fallback)
    codec = Codec(0)
    try:
        codec._concat_per_record = codec._padded_per_record = lambda *a, **k: pytest.fail("per-record fallback")
        got, _ = codec.decode_predict_responses_concat(recs[:3], ["v"])
        assert got["v"].tobytes() == np.concatenate([vals] * 3).tobytes()
        two = [D.entry("v", D.tproto(9, [1, vals.size], V.field(9, [V.encode(vals, 9)]))) + D.mspec(),
               D.entry("v", D.tproto(9, [1, 1000], V.field(9, [V.encode(vals[:1000], 9)]))) + D.mspec()]
        got, shapes, _ = codec.decode_predict_responses_padded(two, ["v"], pad_value=-7)
        want = np.full((2, vals.size), -7, np.int64)
        want[0] = vals
        want[1, :1000] = vals[:1000]
        assert got["v"].tobytes() == want.tobytes() and shapes["v"].tolist() == [[1, vals.size], [1, 1000]]
    finally:
        codec.close()


def straddle_record(dtype, key="v"):
    """One chunk of 1-byte values with a 10-byte varint starting s bytes before window edge s, for s = 1..10, placed as record
    0 of place() (its arena address is 256-byte aligned): (record, values)."""
    for pad in range(0, 16):
        n = 11 * V.DEC_TILE
        probe = record(key + "p" * pad, dtype, n, [b"\x01" * n])
        c0 = chunk_offsets(probe, dtype, [b"\x01" * n])[0]
        if c0 % 16 == 5:
            break
    base = c0 - c0 % 16                                         # the chunk's first window starts here (record offset)
    vals = np.ones(n, dtype=np.int64)
    pos = 0
    out = []
    for s in range(1, 11):
        start = base + s * V.DEC_TILE - s - c0                  # chunk offset of the wide varint
        k = start - pos                                         # 1-byte values before it
        out.append(np.arange(k) % 100 + 1)
        out.append(np.array([-s]))
        pos = start + 10
    used = sum(x.size for x in out)
    out.append(np.full(n - used - 90, 5))
    vals = np.concatenate(out).astype(NP[dtype])
    wire = V.encode(vals, dtype)
    rec = record(key + "p" * pad, dtype, vals.size, [wire])
    assert chunk_offsets(rec, dtype, [wire])[0] == c0
    starts, lens, _ = V.split_varints(wire)
    long_at = c0 + starts[lens == 10]
    assert sorted(((base + (s + 1) * V.DEC_TILE - a) for s, a in enumerate(long_at))) == list(range(1, 11))
    return rec, vals


def test_decode_varints_across_window_edges(dev):
    rec, vals = straddle_record(9)
    # a chunk that ends exactly on a window edge, then one that starts mid-window
    # (record 0 of place() lies 256-byte aligned, so record offsets are arena phases)
    a = np.arange(2 * V.DEC_TILE - 7) % 100
    b = np.arange(300) % 100 + 1
    chunks = [V.encode(a, 9), V.encode(b, 9)]
    for pad in range(16):
        edge = record("w" + "q" * pad, 9, a.size + b.size, chunks)
        c = chunk_offsets(edge, 9, chunks)
        if (c[0] + len(chunks[0]) - (c[0] - c[0] % 16)) % V.DEC_TILE == 0:
            break
    else:
        raise AssertionError("no key length ends the first chunk on a window edge")
    assert c[1] % 16 != 0
    decode_all_routes(dev, [rec], [vals], graph=True)
    decode_all_routes(dev, [edge], [np.concatenate([a, b]).astype(np.int64)])


# ---- errors at the edges ------------------------------------------------------------------------------------------------
def edge_error_cases():
    """(name, wire, dtype, chunks, n): malformed, out-of-range and wrongly counted outputs at window and group edges."""
    vi = D.vi
    cases = []
    T = V.DEC_TILE
    # The first window of a chunk starts at its address rounded down to 16 bytes, so the first window edge lies 0..15 bytes
    # before chunk offset T, wherever the decoder places the record: positions T-18 .. T+1 put a value on both sides of it.
    # An 11-byte varint across a window edge, and an unterminated last varint at one:
    for at in (T - 18, T - 12, T - 6):
        body = b"\x01" * at + b"\xff" * 10 + b"\x01" + b"\x02" * 100
        cases.append(("eleven_across_%d" % at, 9, [body], at + 1 + 100))
    for end in range(T - 15, T + 1, 3):
        cases.append(("unterminated_%d" % end, 9, [b"\x01" * (end - 1) + b"\x80"], end))
    # an out-of-range value as the last element of a window and as the first of the next
    for dt in (6, 5, 4, 17):
        lo, hi = V.RANGE[dt]
        for at in range(T - 18, T + 2):
            v = np.ones(T + 64, dtype=np.int64)
            v[at] = hi + 1 if at % 2 else lo - 1 if lo < 0 else hi + 1
            cases.append(("range_%s_%d" % (V.NAMES[dt], at), dt, [V.encode(v, 3)], v.size))
    # a count one off at one group of elements, strict and tolerant; and the three errors combined
    big = np.ones(V.ENC_GROUP_ELEMS, dtype=np.int64)
    big[0] = 300                                  # two bytes: the record holds as many bytes as elements for the short count
    for n in (V.ENC_GROUP_ELEMS - 1, V.ENC_GROUP_ELEMS + 1):
        cases.append(("count_%d" % n, 3, [V.encode(big[:V.ENC_GROUP_ELEMS], 3)], n))
    eleven_300 = b"\xac\x82" + b"\x80" * 8 + b"\x00"
    cases.append(("parse_range", 6, [vi(1) + eleven_300], 2))
    cases.append(("range_count", 6, [vi(1) + vi(2) + vi(300)], 4))
    cases.append(("parse_range_count", 6, [vi(300) + vi(1) + b"\xff" * 10 + b"\x01"], 7))
    cases.append(("range_count_window", 5, [V.encode(np.r_[np.ones(T - 8), 40000, np.ones(50)].astype(np.int64), 3)], T + 40))
    return [(name, record("x", dt, n, chunks), dt, chunks, n) for name, dt, chunks, n in cases]


def _ref_outcome(dt, chunks, n, strict):
    vals, st = V.decode(chunks, dt, n, tolerant=not strict)
    return ("ok", {"x": vals.astype(NP[dt]).tobytes()}) if st == V.OK else ("raise", V.EXCEPTION[st])


def _codec_outcome(codec, wire, strict):
    try:
        arrays, _ = codec.decode_predict_responses([wire], strict=strict)[0]
        return "ok", {k: v.tobytes() for k, v in arrays.items()}
    except (DecodeError, ValueError, OverflowError) as e:
        return "raise", type(e).__name__


@pytest.mark.parametrize("strict", [True, False])
def test_decode_errors_at_the_edges_in_the_reference_order(strict):
    fresh, warmed = Codec(0), Codec(0)
    try:
        warmed.decode_predict_responses([wire_oracle.build_predict_response([("ids", np.arange(9, dtype=np.int64))])])
        assert warmed._seen_varints
        for name, wire, dt, chunks, n in edge_error_cases():
            want = _ref_outcome(dt, chunks, n, strict)
            fresh._seen_varints = False       # the two-phase route
            assert _codec_outcome(fresh, wire, strict) == want, (name, "two-phase")
            assert _codec_outcome(warmed, wire, strict) == want, (name, "single-launch")
    finally:
        fresh.close()
        warmed.close()


def test_the_varint_switch_adds_three_launches(dev):
    rng = np.random.default_rng(23)
    vals = mixed(9, 5000, rng)
    recs = [record("v", 9, vals.size, [V.encode(vals, 9)])] * 2
    used = {}
    for on in (0, 1):
        s = Single(dev, recs, varints=on)
        try:
            s.run()
            before = s.launches()
            s.run()
            used[on] = s.launches() - before
        finally:
            s.close()
    assert used[1] == used[0] + 3
