"""Packed-varint outputs decoded by the single-launch decode (b200tfs_set_decode_varints).

Every value is checked bit-exact against the two-phase route (b200tfs_parse_responses + b200tfs_unpack_outputs with
dst_dtype NULL, which the header names as the reference for this switch) and, where the oracle decodes the record, against
oracle/wire_oracle.  Every slot byte outside the laid-out ranges must keep the caller's 0xEE fill.
"""
import ctypes as C

import numpy as np
import pytest
from google.protobuf.message import DecodeError

import decode_mutants as D
from devutil import Dev
from min_tfs_client import _native as N
from min_tfs_client.codec import Codec
from oracle import ref_port, wire_oracle

pytestmark = pytest.mark.gpu

K = N.FUSED_MAX_OUTPUTS
FILL = 0xEE
# dtype -> (TensorProto value field, element size in memory, numpy type of the memory, value range)
VARINT = {
    6: (7, 1, np.int8, (-128, 127)), 5: (7, 2, np.int16, (-32768, 32767)), 3: (7, 4, np.int32, (-2**31, 2**31 - 1)),
    4: (7, 1, np.uint8, (0, 255)), 17: (7, 2, np.uint16, (0, 65535)), 22: (16, 4, np.uint32, (0, 2**32 - 1)),
    9: (10, 8, np.int64, (-2**63, 2**63 - 1)), 23: (17, 8, np.uint64, (0, 2**64 - 1)), 10: (11, 1, np.bool_, (0, 1)),
    19: (13, 2, np.uint16, (0, 65535)), 14: (13, 2, np.uint16, (0, 65535)),
}


@pytest.fixture(scope="module")
def dev():
    d = Dev()
    yield d
    d.close()


def fld(field, payload):
    return D.vi((field << 3) | 2) + D.vi(len(payload)) + payload


def output(key, dtype, dims, chunks, unpacked=None):
    """One map entry; `chunks`: packed occurrences of the value field (bytes each); `unpacked`: values as single elements."""
    field = VARINT[dtype][0] if dtype in VARINT else 5
    body = b"".join(fld(field, c) for c in chunks)
    if unpacked is not None:
        body += b"".join(D.vi(field << 3) + D.vi(int(v)) for v in unpacked)
    return D.entry(key, D.tproto(dtype, dims, body))


def response(*entries):
    return b"".join(entries) + D.mspec()


def sample(dtype, n, rng):
    """Values of `dtype` that give varints of every length the dtype can have (1..10 bytes for the signed 32/64-bit ones)."""
    lo, hi = VARINT[dtype][3]
    edges = [lo, hi, 0, 1, -1 if lo < 0 else 2] + [(1 << (7 * k)) - 1 for k in range(1, 10)] + [1 << (7 * k) for k in range(1, 10)]
    edges = [v for v in edges if lo <= v <= hi]
    if dtype == 9:
        body = rng.integers(lo, hi, n, dtype=np.int64, endpoint=True)
    elif dtype == 23:
        body = rng.integers(0, 2**64 - 1, n, dtype=np.uint64, endpoint=True)
    else:
        body = rng.integers(lo, hi, n, endpoint=True)
    vals = [int(v) for v in body]
    vals[: min(n, len(edges))] = edges[: min(n, len(edges))]
    return vals


def packed(vals):
    return b"".join(D.vi(v) for v in vals)


def split(raw_vals, parts):
    """Packed chunks of the values, split over `parts` occurrences at element boundaries."""
    cut = np.linspace(0, len(raw_vals), parts + 1).astype(int)
    return [packed(raw_vals[cut[i]: cut[i + 1]]) for i in range(parts)]


def place(recs, align=256):
    offs, cur = [], 0
    for i, r in enumerate(recs):
        cur = (cur + align - 1) // align * align + (i * 7) % 64
        offs.append(cur)
        cur += len(r)
    arena = np.zeros(cur + 256, dtype=np.uint8)
    for o, r in zip(offs, recs):
        arena[o: o + len(r)] = np.frombuffer(r, dtype=np.uint8)
    n = len(recs)
    return arena, (C.c_uint64 * n)(*offs), (C.c_uint64 * n)(*[len(r) for r in recs])


def stride_for(recs):
    return (max(len(r) for r in recs) * 9 + 256 * (K + 1) + 255) & ~255


class Single:
    """The single-launch decode of a batch on a fresh context, with the switches given."""

    def __init__(self, dev, recs, stride=None, varints=1, cast=0):
        self.dev, self.recs = dev, recs
        self.stride = stride or stride_for(recs)
        self.arena, self.off, self.ln = place(recs)
        self.ctx = C.c_void_p()
        N.check(dev.lib.b200tfs_create(0, C.byref(self.ctx)))
        N.check(dev.lib.b200tfs_set_decode_varints(self.ctx, varints))
        N.check(dev.lib.b200tfs_set_decode_cast(self.ctx, cast))
        self.arena_dev = dev.upload(self.arena)
        self.dst = dev.malloc(len(recs) * self.stride)

    def close(self):
        self.dev.lib.b200tfs_destroy(self.ctx)
        for p in (self.arena_dev, self.dst):
            self.dev.lib.b200tfs_free(self.dev.ctx, C.c_void_p(p))
            self.dev.allocs.remove(p)

    def fill(self):
        N.check(self.dev.lib.b200tfs_memset(self.ctx, self.dst, FILL, len(self.recs) * self.stride))

    def launches(self):
        v = C.c_uint64()
        N.check(self.dev.lib.b200tfs_kernel_launches(self.ctx, C.byref(v)))
        return v.value

    def stats(self):
        v = [C.c_uint64() for _ in range(3)]
        N.check(self.dev.lib.b200tfs_decode_stats(self.ctx, *[C.byref(x) for x in v]))
        return tuple(x.value for x in v)

    def run(self):
        self.fill()
        N.check(self.dev.lib.b200tfs_decode_responses(self.ctx, self.arena_dev, len(self.recs), self.off, self.ln, self.dst, self.stride))
        return self.results(self.download())

    def download(self):
        out = np.empty(len(self.recs) * self.stride, dtype=np.uint8)
        N.check(self.dev.lib.b200tfs_memcpy_d2h(self.ctx, out.ctypes.data, self.dst, out.nbytes))
        return out

    def results(self, slots):
        n = len(self.recs)
        outs, n_outs, specs, st = (N.Output * (n * K))(), (C.c_int32 * n)(), (N.ModelSpec * n)(), (C.c_int32 * n)()
        N.check(self.dev.lib.b200tfs_decode_results(self.ctx, n, outs, n_outs, specs, st))
        return outs, list(n_outs), list(st), slots


def two_phase(dev, recs):
    """Table and unpacked values of every output by the two-phase route: {(r, k): (status, bytes)} plus the tables."""
    arena, off, ln = place(recs)
    arena_dev = dev.upload(arena)
    n = len(recs)
    outs, n_outs, specs, st = (N.Output * (n * 16))(), (C.c_int32 * n)(), (N.ModelSpec * n)(), (C.c_int32 * n)()
    N.check(dev.lib.b200tfs_parse_responses(dev.ctx, arena_dev, n, off, ln, 16, outs, n_outs, specs, st))
    which, at, total = [], [], 0
    for r in range(n):
        if st[r] != N.OK:
            continue
        for k in range(n_outs[r]):
            o = outs[r * 16 + k]
            if o.status != N.OK or not o.n_elems or int(o.dtype) not in VARINT:
                continue
            which.append((r, k))
            at.append(total)
            total = (total + int(o.dst_bytes) + 255) & ~255
    got = {}
    if which:
        m = len(which)
        p = dev.malloc(total)
        sel = (N.Output * m)(*[outs[r * 16 + k] for r, k in which])
        s = (C.c_int32 * m)()
        N.check(dev.lib.b200tfs_unpack_outputs(dev.ctx, arena_dev, m, sel, (C.c_uint64 * m)(*[off[r] for r, _ in which]),
                                               (C.c_void_p * m)(*[p + a for a in at]), None, s))
        back = dev.download(p, total)
        for j, (r, k) in enumerate(which):
            got[(r, k)] = (s[j], back[at[j]: at[j] + int(sel[j].dst_bytes)].tobytes())
        dev.lib.b200tfs_free(dev.ctx, C.c_void_p(p))
        dev.allocs.remove(p)
    dev.lib.b200tfs_free(dev.ctx, C.c_void_p(arena_dev))
    dev.allocs.remove(arena_dev)
    return got, list(st), list(n_outs)


def check_against_two_phase(dev, recs, res, stride, expect_statuses=None):
    """Statuses and values equal the two-phase route's; OK records' slot bytes outside the decoded ranges keep the fill."""
    outs, n_outs, st, slots = res
    want, want_st, want_n = two_phase(dev, recs)
    seen = {}
    for r in range(len(recs)):
        keep = np.ones(stride, dtype=bool)
        if st[r] == N.OK:
            assert n_outs[r] == want_n[r]
            for k in range(n_outs[r]):
                o = outs[r * K + k]
                if (r, k) in want:
                    ws, wb = want[(r, k)]
                    assert o.flags & N.OF_DEVICE_VARINT, (r, k)
                    assert o.status == ws, (r, k, o.status, ws)
                    seen[(r, k)] = o.status
                    if ws == N.OK:
                        a = int(o.dst_off)
                        assert a % 256 == 0 and a + int(o.dst_bytes) <= stride
                        assert slots[r * stride + a: r * stride + a + int(o.dst_bytes)].tobytes() == wb, (r, k)
                    if o.status != N.E_SIZE:
                        keep[int(o.dst_off): int(o.dst_off) + int(o.dst_bytes)] = False
                elif o.status == N.OK and o.n_elems and int(o.dtype) in (1, 2, 8, 18):
                    keep[int(o.dst_off): int(o.dst_off) + int(o.dst_bytes)] = False
        assert (slots[r * stride: (r + 1) * stride][keep] == FILL).all(), r
    if expect_statuses is not None:
        assert sorted(seen.values()) == sorted(expect_statuses)
    return seen


def every_dtype_records(rng, n_each=300):
    recs = []
    for dt in VARINT:
        for n in (0, 1, n_each):
            vals = sample(dt, n, rng)
            raw = [v & ((1 << 64) - 1) if v < 0 else v for v in vals]
            recs.append(response(output("scores", 1, [3], [np.float32([1, 2, 3]).tobytes()]),
                                 output("v", dt, [n], split(raw, 1 + n % 8) if n else [])))
    return recs


def test_every_dtype_and_varint_length_matches_two_phase_and_oracle(dev):
    rng = np.random.default_rng(1)
    recs = every_dtype_records(rng)
    s = Single(dev, recs)
    try:
        for _ in range(2):     # the second launch takes the templates the first one left
            res = s.run()
            seen = check_against_two_phase(dev, recs, res, s.stride)
            assert seen and all(v == N.OK for v in seen.values())
        outs, n_outs, st, slots = res
        for r, rec in enumerate(recs):
            ref = wire_oracle.decode_predict_response(rec, strict=False)
            o = outs[r * K + 1]
            if o.n_elems and int(o.dtype) in VARINT:
                a = r * s.stride + int(o.dst_off)
                got = slots[a: a + int(o.dst_bytes)].tobytes()
                assert got == np.ascontiguousarray(ref["v"]).tobytes(), r
    finally:
        s.close()


def test_eight_outputs_mixed_and_a_million_elements(dev):
    rng = np.random.default_rng(2)
    big = sample(9, 1 << 20, rng)
    raw = [v & ((1 << 64) - 1) for v in big]
    ents = [output("big", 9, [1 << 20], split(raw, 8))]
    for i, dt in enumerate((6, 10, 23, 19, 22, 3)):
        v = sample(dt, 257, rng)
        ents.append(output(f"o{i}", dt, [257], [packed([x & ((1 << 64) - 1) for x in v])]))
    ents.append(output("f", 1, [5], [np.arange(5, dtype=np.float32).tobytes()]))
    rec = response(*ents)
    s = Single(dev, [rec, rec])
    try:
        for _ in range(2):
            seen = check_against_two_phase(dev, [rec, rec], s.run(), s.stride)
            assert len(seen) == 14 and all(v == N.OK for v in seen.values())
    finally:
        s.close()


def test_errors_are_reported_per_output(dev):
    good = packed([1, 2, 300])
    recs = [
        response(output("shape", 9, [4], [good])),                                   # 3 values for 4 elements
        response(output("parse", 9, [4], [packed([1, 2]) + b"\xff" * 10 + b"\x01"])),   # an 11-byte varint, count wrong too
        response(output("range", 6, [3], [good])),                                   # int_val 300 as DT_INT8
        response(output("rows", 3, [3], [], unpacked=[5, 6, 7])),                     # unpacked elements
        response(output("ok", 3, [3], [good]), output("ok2", 10, [2], [b"\x01\x00"])),
    ]
    s = Single(dev, recs)
    try:
        res = s.run()
        # (the two-phase route gathers the unpacked row itself: compared separately below)
        seen = check_against_two_phase(dev, recs[:3] + recs[4:], _sub(res, [0, 1, 2, 4], s.stride), s.stride)
        outs = res[0]
        assert outs[0].status == N.E_SHAPE and outs[K].status == N.E_PARSE and outs[2 * K].status == N.E_RANGE
        assert outs[3 * K].status == N.E_NONCANONICAL and outs[3 * K].flags & N.OF_DEVICE_VARINT
        assert outs[4 * K].status == N.OK and outs[4 * K + 1].status == N.OK and seen
        # the row of unpacked elements, finished by b200tfs_unpack_outputs from the same table entry
        o = outs[3 * K]
        o.status = N.OK
        p = dev.malloc(12)
        st = (C.c_int32 * 1)()
        N.check(dev.lib.b200tfs_unpack_outputs(s.ctx, s.arena_dev, 1, (N.Output * 1)(o), (C.c_uint64 * 1)(s.off[3]), (C.c_void_p * 1)(p), None, st))
        assert st[0] == N.OK and dev.download(p, 12, np.int32).tolist() == [5, 6, 7]
    finally:
        s.close()
    # a slot too small for the varint range: E_SIZE, nothing stored
    rec = response(output("f", 1, [64], [np.zeros(64, np.float32).tobytes()]), output("ids", 9, [200], [packed(range(200))]))
    s = Single(dev, [rec], stride=512)
    try:
        outs, n_outs, st, slots = s.run()
        assert st[0] == N.OK and outs[0].status == N.OK and outs[1].status == N.E_SIZE
        assert (slots[256:] == FILL).all()
    finally:
        s.close()


def _sub(res, idx, stride):
    outs, n_outs, st, slots = res
    o2 = (N.Output * (len(idx) * K))()
    for j, r in enumerate(idx):
        for k in range(K):
            o2[j * K + k] = outs[r * K + k]
    parts = np.concatenate([slots[r * stride: (r + 1) * stride] for r in idx])
    return o2, [n_outs[r] for r in idx], [st[r] for r in idx], parts


def test_switch_off_leaves_varint_outputs_tabulated_only(dev):
    rng = np.random.default_rng(3)
    recs = every_dtype_records(rng, 40)
    s = Single(dev, recs, varints=0)
    try:
        outs, n_outs, st, slots = s.run()
        for r in range(len(recs)):
            keep = np.ones(s.stride, dtype=bool)
            for k in range(n_outs[r]):
                o = outs[r * K + k]
                assert not o.flags & N.OF_DEVICE_VARINT
                if int(o.dtype) == 1:
                    assert o.dst_off == 0
                    keep[: int(o.dst_bytes)] = False
                else:
                    assert o.status == N.OK
            assert (slots[r * s.stride: (r + 1) * s.stride][keep] == FILL).all()
    finally:
        s.close()


def test_host_wire_routes_and_the_narrowing_batch(dev):
    rng = np.random.default_rng(4)
    ids = [int(v) for v in rng.integers(0, 50000, 4096)]
    rec = response(output("ids", 9, [8, 512], [packed(ids)]), output("scores", 1, [8, 512], [rng.standard_normal(4096).astype(np.float32).tobytes()]))
    recs = [rec] * 4
    want = np.array(ids, dtype=np.int64).tobytes()
    s = Single(dev, recs)
    try:
        stride = s.stride
        buf = np.frombuffer(b"".join(recs), dtype=np.uint8).copy()
        off = (C.c_uint64 * 4)(*[i * len(rec) for i in range(4)])
        ln = (C.c_uint64 * 4)(*[len(rec)] * 4)
        hp = C.c_void_p()
        N.check(dev.lib.b200tfs_host_alloc(4 * stride, C.byref(hp)))
        try:
            for direct in (True, False):
                if not direct:
                    N.check(dev.lib.b200tfs_set_pipeline(s.ctx, 0, 0))
                C.memset(hp, FILL, 4 * stride)
                N.check(dev.lib.b200tfs_decode_responses_host_async(s.ctx, buf.ctypes.data, 4, off, ln, hp, stride))
                outs, n_outs, st, _ = s.results(None)
                host = np.frombuffer((C.c_uint8 * (4 * stride)).from_address(hp.value), dtype=np.uint8)
                for r in range(4):
                    o = outs[r * K]
                    assert st[r] == N.OK and o.status == N.OK and o.flags & N.OF_DEVICE_VARINT
                    a = r * stride + int(o.dst_off)
                    assert host[a: a + len(want)].tobytes() == want
        finally:
            dev.lib.b200tfs_host_free(hp)
    finally:
        s.close()
    # three-launch narrowing batch (>= 4 MiB of records the host has a template for), fp16 on
    big = [rec] * (4 * 1024 * 1024 // len(rec) + 2)
    s = Single(dev, big, cast=19)
    try:
        first = s.run()
        before = s.launches()
        outs, n_outs, st, slots = s.run()
        assert s.launches() - before == 3 + 3       # verify, guarded move, fallback; plan, count, emit
        for r in range(len(big)):
            o = outs[r * K]
            assert st[r] == N.OK and o.status == N.OK
            a = r * s.stride + int(o.dst_off)
            assert slots[a: a + len(want)].tobytes() == want
        assert first[1] == n_outs
    finally:
        s.close()


def test_graph_capture_replays_template_and_walk(dev):
    def rec_of(a, b):
        return response(output("a", 9, [64], [packed(a)]), output("b", 3, [64], [packed(b)]),
                        output("f", 1, [4], [np.ones(4, np.float32).tobytes()]))
    a, b = list(range(64)), list(range(100, 164))     # b: 1- and 2-byte varints
    recs = [rec_of(a, b)] * 3
    s = Single(dev, recs)
    try:
        s.run()
        N.check(dev.lib.b200tfs_sync(s.ctx))
        N.check(dev.lib.b200tfs_capture_begin(s.ctx))
        N.check(dev.lib.b200tfs_decode_responses(s.ctx, s.arena_dev, 3, s.off, s.ln, s.dst, s.stride))
        g = C.c_void_p()
        N.check(dev.lib.b200tfs_capture_end(s.ctx, C.byref(g)))
        # same varint lengths, new values: the template
        a2, b2 = [v ^ 1 for v in a], [v ^ 3 for v in b]
        # other varint lengths in both outputs (one byte longer / shorter): same record length, other framing - the walk
        a3, b3 = [200] + a[1:], b[:-1] + [5]
        for va, vb, path in ((a2, b2, "template"), (a3, b3, "walk")):
            new = [rec_of(va, vb)] * 3
            assert len(new[0]) == len(recs[0])
            arena, _, _ = place(new)
            N.check(dev.lib.b200tfs_memcpy_h2d(s.ctx, s.arena_dev, arena.ctypes.data, arena.nbytes))
            s.fill()
            before = s.stats()
            N.check(dev.lib.b200tfs_graph_launch(s.ctx, g))
            res = s.results(s.download())
            after = s.stats()
            assert (after[2] - before[2] == 3) == (path == "walk"), (path, before, after)
            check_against_two_phase(dev, new, res, s.stride)
            outs = res[0]
            assert all(outs[r * K + k].status == N.OK for r in range(3) for k in range(2))
        N.check(dev.lib.b200tfs_graph_destroy(g))
    finally:
        s.close()


@pytest.mark.parametrize("cast", [0, 19])
def test_mutant_corpus_matches_two_phase(dev, cast):
    recs = []
    for seed, ms in D.corpus():
        if seed.tensor:
            continue
        recs += [m.record for m in ms if len(m.record)]
    recs = [r for r in recs if len(r) < (1 << 16)]
    taken = 0
    for i in range(0, len(recs), 512):
        batch = recs[i: i + 512]
        s = Single(dev, batch, cast=cast)
        try:
            res = s.run()
            outs, n_outs, st, slots = res
            want, want_st, want_n = two_phase(dev, batch)
            for r in range(len(batch)):
                if st[r] != N.OK:
                    continue
                for k in range(n_outs[r]):
                    o = outs[r * K + k]
                    assert o.status != N.E_SIZE, (i + r, k)          # the stride has room for every output
                    if (r, k) not in want:                           # not a varint output the two-phase route decodes
                        assert not o.flags & N.OF_DEVICE_VARINT, (i + r, k)
                        continue
                    ws, wb = want[(r, k)]
                    assert o.flags & N.OF_DEVICE_VARINT and o.status == ws, (i + r, k, o.status, ws)
                    if ws == N.OK:
                        a = r * s.stride + int(o.dst_off)
                        assert slots[a: a + int(o.dst_bytes)].tobytes() == wb
                    taken += 1
        finally:
            s.close()
    assert taken > 1000


def _classify(rng, n=4):
    return [wire_oracle.build_predict_response([("classes", rng.integers(0, 1000, (8, 5)).astype(np.int64)),
                                                ("ids", rng.integers(-5, 50000, (3, 7)).astype(np.int32)),
                                                ("mask", rng.integers(0, 2, 9).astype(bool)),
                                                ("scores", rng.standard_normal((8, 5)).astype(np.float32))]) for _ in range(n)]


def test_python_decode_takes_the_varint_route_after_the_first_response(monkeypatch):
    codec = Codec(0)
    try:
        rng = np.random.default_rng(5)
        wires = _classify(rng)
        calls = []
        real = codec._lib.b200tfs_unpack_outputs_host
        monkeypatch.setattr(codec._lib, "b200tfs_unpack_outputs_host", lambda *a: calls.append(1) or real(*a))
        for strict in (False, True, False):
            got = codec.decode_predict_responses(wires, strict=strict)
            for w, (arrays, _) in zip(wires, got):
                ref = wire_oracle.decode_predict_response(w, strict=strict)
                assert set(arrays) == set(ref)
                for k in ref:
                    assert arrays[k].dtype == ref[k].dtype and arrays[k].shape == ref[k].shape and arrays[k].tobytes() == ref[k].tobytes()
        assert len(calls) == 1            # the first call learnt that these responses carry varint outputs
        assert codec._seen_varints
    finally:
        codec.close()


def _check_oracle(codec, wires, strict=False):
    for w, (arrays, _) in zip(wires, codec.decode_predict_responses(wires, strict=strict)):
        ref = wire_oracle.decode_predict_response(w, strict=strict)
        assert set(arrays) == set(ref)
        for k in ref:
            assert arrays[k].dtype == ref[k].dtype and arrays[k].shape == ref[k].shape and arrays[k].tobytes() == ref[k].tobytes(), k


def test_python_slots_are_sized_from_the_records_of_each_call(monkeypatch):
    """A response whose varints are denser than any seen before still decodes in one launch (its slots are sized from its own
    records); a float-only call after varint traffic keeps the plain stride and leaves the switch off."""
    codec = Codec(0)
    try:
        rng = np.random.default_rng(7)

        def tokens(ids):
            return wire_oracle.build_predict_response([("ids", ids.astype(np.int64)), ("scores", rng.standard_normal((8, 512)).astype(np.float32))])
        sparse = [tokens(rng.integers(0, 50000, (8, 512))) for _ in range(2)]
        dense = [tokens(np.where(rng.random((8, 512)) < 0.95, 0, rng.integers(1, 50000, (8, 512)))) for _ in range(2)]
        label = [wire_oracle.build_predict_response([("label", np.array([3], np.int64)), ("score", np.array([0.5], np.float32))])]
        floats = [wire_oracle.build_predict_response([("scores", rng.standard_normal((64, 1024)).astype(np.float32))]) for _ in range(3)]
        _check_oracle(codec, sparse)
        calls = []
        real = codec._lib.b200tfs_unpack_outputs_host
        monkeypatch.setattr(codec._lib, "b200tfs_unpack_outputs_host", lambda *a: calls.append(1) or real(*a))
        for wires in (dense, label, sparse, dense):
            buf, off, ln = codec._pack_wires(wires)
            stride, on = codec._slot_stride(buf, off, ln)
            assert on and stride >= max(len(w) for w in wires) + 256 * (K + 1)
            _check_oracle(codec, wires)
            _check_oracle(codec, wires, strict=True)
        assert calls == []
        buf, off, ln = codec._pack_wires(floats)
        assert codec._slot_stride(buf, off, ln) == ((max(len(w) for w in floats) + 256 * (K + 1) + 255) & ~255, False)
        _check_oracle(codec, floats)
    finally:
        codec.close()


@pytest.mark.parametrize("strict", [True, False])
def test_python_errors_are_unchanged(strict):
    bad = [
        response(output("x", 9, [4], [packed([1, 2, 3])])),                  # too few values: ValueError / TF padding
        response(output("x", 9, [4], [packed([1, 2]) + b"\xff" * 10 + b"\x01"])),   # malformed varint: DecodeError
        response(output("x", 6, [3], [packed([1, 2, 300])])),                # out of range: OverflowError
        response(output("x", 3, [3], [], unpacked=[5, 6, 7])),               # rows of unpacked elements
        response(output("x", 19, [2], [packed([18688, 1])])),                # DT_HALF: values (strict) or bits
        # more than one error in one output: DecodeError before OverflowError before ValueError
        response(output("x", 6, [2], [packed([1]) + b"\xac\x82" + b"\x80" * 8 + b"\x00"])),   # 11-byte varint reading 300
        response(output("x", 6, [4], [packed([1, 2, 300])])),                # out of range and too few values
        response(output("x", 5, [7], [packed([1, 40000]) + b"\xff" * 10 + b"\x01"])),   # all three
        response(output("x", 4, [3], [packed([256]), packed([1])])),          # out of range in one chunk, count wrong
    ]
    warm = _classify(np.random.default_rng(6), 1)

    def outcome(codec, w):
        if codec is fresh:
            codec._seen_varints = False     # as before this codec saw a varint output: the switch stays off
        try:
            arrays, _ = codec.decode_predict_responses([w], strict=strict)[0]
            return ("ok", {k: (v.dtype.str, v.shape, v.tobytes()) for k, v in arrays.items()})
        except (DecodeError, ValueError, OverflowError, KeyError, TypeError, NotImplementedError) as e:
            return ("raise", type(e).__name__)

    def reference(w):
        try:
            return ("ok", {k: (v.dtype.str, v.shape, v.tobytes()) for k, v in ref_port.decode_predict_response(w).items()})
        except (DecodeError, ValueError, OverflowError) as e:
            return ("raise", type(e).__name__)

    fresh, warmed = Codec(0), Codec(0)
    try:
        warmed.decode_predict_responses(warm)
        assert warmed._seen_varints and not fresh._seen_varints
        for w in bad:
            assert outcome(warmed, w) == outcome(fresh, w), w
            if strict:
                assert outcome(fresh, w) == reference(w), w
    finally:
        fresh.close()
        warmed.close()
