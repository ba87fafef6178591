"""The fixed-width move engine on the device at every source phase, destination phase, tile, round and staged-chunk edge,
compared byte for byte with the oracle (wire_oracle.encode_predict_request for the encodes, decode_predict_response for the
decodes) - never with another route.

Every destination is filled with a canary first; afterwards every byte outside the promised ranges must still hold it.  Every
test asserts, through the geometry model of tests/move_ref.py fed with the real device addresses, that it reached the edges it
is named for: the (source phase k, destination phase) pairs per vector body, tile and round counts, staged chunk counts, last
chunk sizes and the waits on barrier parity 1.
"""
import ctypes as C
import os

import ml_dtypes
import numpy as np
import pytest

import cast_sweep
import move_ref as M
from devutil import Dev, tensor_struct
from min_tfs_client import _native as N
from oracle import wire_oracle
from test_device_api_gpu import _response_with_chunks, _vi

pytestmark = pytest.mark.gpu

CANARY = 0xA7


@pytest.fixture()
def fresh():
    """fresh(tile_bytes): a new context created with B200TFS_TILE_BYTES set (None: unset); the variable is restored at once
    and every context is closed at teardown."""
    made = []

    def make(tile_bytes=None):
        old = os.environ.get("B200TFS_TILE_BYTES")
        if tile_bytes is None:
            os.environ.pop("B200TFS_TILE_BYTES", None)
        else:
            os.environ["B200TFS_TILE_BYTES"] = str(tile_bytes)
        try:
            d = Dev(0)
        finally:
            if old is None:
                os.environ.pop("B200TFS_TILE_BYTES", None)
            else:
                os.environ["B200TFS_TILE_BYTES"] = old
        made.append(d)
        return d

    yield make
    for d in made:
        d.close()


def canary_buffer(dev, nbytes):
    p = dev.malloc(nbytes)
    N.check(dev.lib.b200tfs_memset(dev.ctx, p, CANARY, nbytes))
    return p


def same_image(got, want, what):
    """Whole buffers equal (the promised ranges hold the reference bytes, every other byte the canary); on a difference,
    say where."""
    if not np.array_equal(got, want):
        bad = np.flatnonzero(got != want)
        pytest.fail(f"{what}: {bad.size} bytes differ, first at {int(bad[0])}: got {got[bad[0]: bad[0] + 8].tobytes().hex()} "
                    f"want {want[bad[0]: bad[0] + 8].tobytes().hex()}")


def patterns(nbytes, seed):
    """nbytes of float32 specials (sNaN / qNaN / inf / denormals / -0) mixed with random bits, the specials at the head, at
    every 16-byte block and in the tail."""
    bits = np.resize(np.roll(cast_sweep.f32_patterns()[:4096], seed), (nbytes + 3) // 4).copy()
    bits[1::7] = 0x7F800001 + (np.arange(bits[1::7].size, dtype=np.uint32) % 0x3FFFFF)   # sNaNs throughout
    return bits.view(np.uint8)[:nbytes].copy()


def edge_lengths(tile, esz, small=True):
    """Byte lengths around every edge of a tile of `tile` bytes, rounded down to whole elements of esz bytes."""
    want = {esz, 15, 16, 17, tile - 17, tile - 1, tile + 1, tile + 17, tile + 16 * 1024 - 16, tile + 16 * 1024 + 16,
            2 * tile - 16, 2 * tile + 16, 3 * tile + 16}
    if small:
        want |= {M.K_SMALL_MAX - 1, M.K_SMALL_MAX, M.K_SMALL_MAX + 1}
    return sorted({(n // esz) * esz for n in want if n // esz})


# ---- E1: encode from device pointers --------------------------------------------------------------------------------------
# (name, numpy dtype, tensor flags, op, wire dtype) - integers travel as tensor_content, float32 either quieted (QUIET_SRC,
# from the source's 4-byte elements) or kept (KEEP_SNAN: a plain copy), float16 widened to DT_FLOAT (H2F)
ENCODE_CASES = [
    ("int8", np.int8, N.F_TENSOR_CONTENT, M.COPY, None), ("uint8", np.uint8, N.F_TENSOR_CONTENT, M.COPY, None),
    ("int16", np.int16, N.F_TENSOR_CONTENT, M.COPY, None), ("uint16", np.uint16, N.F_TENSOR_CONTENT, M.COPY, None),
    ("int32", np.int32, N.F_TENSOR_CONTENT, M.COPY, None), ("int64", np.int64, N.F_TENSOR_CONTENT, M.COPY, None),
    ("float64", np.float64, 0, M.COPY, None), ("complex64", np.complex64, 0, M.COPY, None),
    ("complex128", np.complex128, 0, M.COPY, None), ("f32_keep_snan", np.float32, N.F_KEEP_SNAN, M.COPY, None),
    ("f32_quiet", np.float32, 0, M.QUIET_SRC, None), ("bool", np.bool_, 0, M.BOOL, None),
    ("f16_to_f32", np.float16, 0, M.H2F, np.float32),
]


def encode_batch(dev, reqs, flags, wire_dtype=None):
    """reqs: [(inputs [(key, array, device pointer)])], one encode call into a canary-filled arena.  Returns (arena image,
    arena pointer, rec_off, rec_len)."""
    keep, rq = [], []
    for inputs in reqs:
        ts = []
        for k, a, p in inputs:
            t, dims = tensor_struct(p, a, key=k.encode(), flags=flags, wire_dtype=wire_dtype)
            keep.append(dims)
            ts.append(t)
        arr = (N.Tensor * len(ts))(*ts)
        keep.append(arr)
        N.check(dev.lib.b200tfs_measure(dev.ctx, len(ts), arr))
        rq.append(N.Request(model_name=b"m", model_name_len=1, has_version=1, order=N.ORDER_UPB, version=1, n_inputs=len(ts),
                            flags=0, inputs=arr))
    n = len(rq)
    rq = (N.Request * n)(*rq)
    need = C.c_uint64()
    N.check(dev.lib.b200tfs_request_arena_size(n, rq, C.byref(need)))
    arena = canary_buffer(dev, need.value)
    off, ln = (C.c_uint64 * n)(), (C.c_uint64 * n)()
    N.check(dev.lib.b200tfs_encode_requests(dev.ctx, n, rq, arena, need.value, off, ln))
    return dev.download(arena, need.value), arena, list(off), list(ln)


class Sweep:
    """The outcome of encode_sweep: geometries of the tested payloads that took tiles, and what the plan image of each
    encode call must have held (tiled payloads, and an upper bound of its small items and header blob)."""

    def __init__(self):
        self.geos, self.calls = [], []

    def plan_bounds(self):
        """[(lower, upper)] bytes of each call's plan image: the MoveItems alone, and everything it can hold."""
        return [(M.plan_image(items, 0, 0, 0), M.plan_image(items, tiles, smalls, blob)) for items, tiles, smalls, blob in self.calls]


def encode_sweep(dev, name, np_dt, flags, op, lengths, seed, wire_dt=None, per_call=None, sweep=None, companion=True):
    """Every element-aligned source phase x every length, each tested input ("t...") behind a larger companion ("c...", the
    record's largest payload, which the encode places 128-byte aligned) with random key lengths, so that the tested payload's
    destination phase moves independently of its source phase.  One encode call for the whole sweep (per_call: that many requests per call).  Compared with the oracle inside a canary.
    companion=False: the tested payload is the record's largest, its destination 128-byte aligned."""
    rng = np.random.default_rng(seed)
    esz = np.dtype(np_dt).itemsize
    sw = sweep or Sweep()
    reqs, tested = [], []
    i = 0
    for n in lengths:
        phases = range(0, 16, esz) if n <= 1 << 20 else (0, 16 - esz)
        for shift in [s for s in phases for _ in range(esz if M.K_SMALL_MAX < n <= 1 << 20 else 1)]:
            raw = rng.integers(0, 256, n, dtype=np.uint8) if np_dt is np.bool_ else patterns(n, i)
            comp = rng.integers(0, 256, n + 4096 + esz, dtype=np.uint8)[: (n + 4096) // esz * esz]
            comp = comp.view(np.bool_ if np_dt is np.bool_ else np_dt)
            a = raw.view(np.bool_) if np_dt is np.bool_ else raw.view(np_dt)
            buf = np.zeros(n + 32, np.uint8)
            buf[shift: shift + n] = raw
            p = dev.upload(buf)
            assert p % 256 == 0
            inputs = [("c" * int(rng.integers(1, 4)), comp, dev.upload(comp)), ("t" * int(rng.integers(1, 17)), a, p + shift)]
            if not companion:
                inputs = inputs[1:]
            reqs.append(inputs)
            tested.append((a, raw, p + shift))
            i += 1
    step = per_call or len(reqs)
    kw = {"tensor_content": bool(flags & N.F_TENSOR_CONTENT), "keep_snan": bool(flags & N.F_KEEP_SNAN)}
    if wire_dt:
        kw["wire_dtype"] = wire_dt
    for c0 in range(0, len(reqs), step):
        part = reqs[c0: c0 + step]
        image, arena, off, ln = encode_batch(dev, part, flags, {np.float32: 1}.get(wire_dt))
        want_img = np.full(image.size, CANARY, np.uint8)
        items = tiles = smalls = blob = 0
        for r, inputs in enumerate(part):
            a, raw, src = tested[c0 + r]
            want = wire_oracle.encode_predict_request("m", 1, [(k, x) for k, x, _ in inputs], **kw)
            want_img[off[r]: off[r] + len(want)] = np.frombuffer(want, np.uint8)
            assert ln[r] == len(want), (name, r)
            body = M.out_bytes(op, raw.tobytes())
            large = [len(M.out_bytes(op, x.tobytes())) for _, x, _ in inputs]
            items += sum(x > M.K_SMALL_MAX for x in large)
            tiles += sum(M.tiles_for(x, 2048) for x in large if x > M.K_SMALL_MAX)
            smalls += 2 * len(inputs) + 2
            blob += len(want) - sum(x for x in large if x > M.K_SMALL_MAX)
            if M.route(len(body)) == "tile":
                at = want.find(body)
                assert at > 0 and want.find(body, at + 1) < 0, (name, r)
                sw.geos.append(M.Geometry(src, arena + off[r] + at, len(body), op))
        sw.calls.append((items, tiles, smalls, blob))
        same_image(image, want_img, name)
    return sw


@pytest.mark.parametrize("case", ENCODE_CASES, ids=[c[0] for c in ENCODE_CASES])
def test_encode_from_device_at_every_source_and_destination_phase(fresh, case):
    """E1: one encode call per case over every element-aligned source phase and the lengths around the warp / tile, tile,
    round and 2- / 3-tile edges and one of 3 MiB, each payload behind a companion input so that its destination is not
    16-byte aligned.  The call's plan image is far above kInlinePlanBytes: move_kernel reads it from device memory."""
    name, np_dt, flags, op, wire_dt = case
    esz = np.dtype(np_dt).itemsize
    dev = fresh()
    sw = encode_sweep(dev, name, np_dt, flags, op, edge_lengths(32768, esz) + [(3 << 20) + 3 * esz], esz, wire_dt)
    geos = sw.geos
    vpt = 2048                                               # 32 KB encode tiles: the large payloads of the sweep ask for the cap
    assert {g.src & 15 for g in geos} == set(range(0, 16, esz)), name
    assert {g.dphase for g in geos} == set(range(16)), name
    assert all(not M.inline_plan(lo) for lo, _ in sw.plan_bounds())
    fast = [g for g in geos if g.fast]
    if op == M.H2F:
        # body_widen needs both sides 16-byte aligned, else the byte generator: a record whose widened payload is its largest
        # (placed 128-byte aligned) from an aligned source takes it, over 1 to 7 tiles of two rounds of units each
        assert all(g.fast == (g.src % 16 == 0 and g.dphase == 0) for g in geos) and None in {g.body() for g in geos}
        alone = encode_sweep(dev, name, np_dt, flags, op, edge_lengths(32768, esz) + [(1 << 20) + 2], 3, wire_dt, companion=False).geos
        assert "widen" in {g.body() for g in alone} and any(len(g.tiles(vpt)) >= 3 for g in alone if g.fast)
        return
    assert {g.body() for g in fast} >= {"aligned", "shifted0", "shifted1", "shifted2", "shifted3"}, name
    assert any(len(g.tiles(vpt)) >= 3 for g in fast) and any(g.tail and g.head for g in fast)
    assert max(g.n_out for g in geos) > 3 << 20
    if op == M.QUIET_SRC:
        assert all(g.fast for g in geos)                     # float32 sources are 4-byte aligned: the PRE variant


def test_encode_plan_in_the_parameters(fresh):
    """E1, plan placement: one request per call (int8 at every source phase, float32 quieting, bool): each call's plan image
    fits kInlinePlanBytes and travels in the kernel parameters (move_kernel_inline)."""
    dev = fresh()
    sw = Sweep()
    for name, np_dt, flags, op, wire_dt in (ENCODE_CASES[0], ENCODE_CASES[10], ENCODE_CASES[11]):
        esz = np.dtype(np_dt).itemsize
        encode_sweep(dev, name, np_dt, flags, op, [n // esz * esz for n in (M.K_SMALL_MAX + 4, 32768 + 20, 3 * 32768 + 16)], 5,
                     per_call=1, sweep=sw)
    assert len(sw.calls) >= 16 * 3 and all(M.inline_plan(hi) for _, hi in sw.plan_bounds())
    assert {g.src & 15 for g in sw.geos} == set(range(16)) and {g.dphase for g in sw.geos} == set(range(16))


@pytest.mark.parametrize("tile_bytes", [32, 64, 96, 65536])
def test_encode_small_and_override_tiles(fresh, tile_bytes):
    """E1 under B200TFS_TILE_BYTES: tiles of 2, 4 and 6 vectors put hundreds of tile edges inside small payloads; 64 KB tiles
    run body_aligned and body_shifted_q for two rounds."""
    dev = fresh(tile_bytes)
    vpt = M.pick_vec_per_tile(132, 1, 32768, override=tile_bytes)
    lengths = [M.K_SMALL_MAX + 1, 4099, 65536 + 17, 65536 + 16 * 2048 + 3] if tile_bytes == 65536 else [M.K_SMALL_MAX + 1, 2100, 4099]
    seen = set()
    for name, np_dt, flags, op, wire_dt in (ENCODE_CASES[0], ENCODE_CASES[10], ENCODE_CASES[11]):
        esz = np.dtype(np_dt).itemsize
        for g in encode_sweep(dev, name, np_dt, flags, op, [n // esz * esz for n in lengths], 7).geos:
            for t, v0, n, rounds in g.tiles(vpt):
                seen.add((g.body(), rounds))
    if tile_bytes == 65536:
        assert ("aligned", 2) in seen and any(b and b.startswith("shifted") and r == 2 for b, r in seen), seen
    else:
        assert {b for b, _ in seen} >= {"aligned", "shifted1", "shifted3"}


@pytest.mark.parametrize("case", [ENCODE_CASES[6], ENCODE_CASES[10], ENCODE_CASES[11], ENCODE_CASES[12]],
                         ids=["float64", "f32_quiet", "bool", "f16_to_f32"])
def test_host_encode_from_misaligned_host_buffers(fresh, case):
    """E2: b200tfs_encode_requests_host_async from host arrays at every element-aligned offset (np.frombuffer(..., offset=s)).
    The staging copy does not keep the host's phase: every host tensor is copied to a 256-byte boundary of the staging buffer
    (stage_tensors), so on the device the source is 16-byte aligned whatever the host offset, and the destination phase alone
    decides the body.  Compared with the oracle."""
    from test_host_pipeline_gpu import _encode_host
    name, np_dt, flags, op, wire_dt = case
    esz = np.dtype(np_dt).itemsize
    dev = fresh()
    rng = np.random.default_rng(13)
    batch, hits = [], set()
    for n in (M.K_SMALL_MAX + esz, 32768 + 16 + esz, (1 << 20) + 3 * esz):
        for s in range(0, 16, esz):
            host = np.zeros(n + 32, np.uint8)
            host[s: s + n] = rng.integers(0, 256, n, dtype=np.uint8) if np_dt is np.bool_ else patterns(n, s)
            a = np.frombuffer(host.data, dtype=np_dt, count=n // esz, offset=s)
            assert a.ctypes.data % 16 == s
            comp = np.frombuffer(rng.integers(0, 256, n + 4096, dtype=np.uint8).tobytes(), dtype=np_dt)
            batch.append(("m", 1, [("c" * (1 + s % 3), comp), ("t" * (1 + (5 * s) % 16), a)]))
            hits.add(s)
    wires = _encode_host(dev, batch, pinned_inputs=False, wire_dtypes={(b, k): 1 for b in range(len(batch)) for k in range(2)} if wire_dt else None)
    kw = {"wire_dtype": wire_dt} if wire_dt else {}
    for b, (model, version, inputs) in enumerate(batch):
        assert wires[b] == wire_oracle.encode_predict_request(model, version, inputs, **kw), (name, b)
    assert hits == set(range(0, 16, esz))


# ---- D1: two-phase decode (parse + unpack) at every source x destination phase ---------------------------------------------
D1_CASES = [  # (name, array builder(nbytes, seed), build kw, dst dtype for the unpack (0: the wire's), op, element bytes in/out)
    ("uint8_content", lambda n, s: patterns(n, s), {"tensor_content": True}, 0, M.COPY, 1, 1),
    ("int8_content", lambda n, s: patterns(n, s).view(np.int8), {"tensor_content": True}, 0, M.COPY, 1, 1),
    ("float_val", lambda n, s: patterns(n, s).view(np.float32), {"keep_snan": True}, 0, M.QUIET_DST, 4, 4),
    ("double_val", lambda n, s: patterns(n, s).view(np.float64), {}, 0, M.COPY, 8, 8),
    ("float_val_to_f16", lambda n, s: patterns(n, s).view(np.float32), {"keep_snan": True}, 19, M.F2H, 4, 2),
    ("float_val_to_bf16", lambda n, s: patterns(n, s).view(np.float32), {"keep_snan": True}, 14, M.F2B, 4, 2),
]
# tensor_content is what TensorFlow's MakeNdarray reads (the oracle's tolerant mode; the reference reads typed fields only)
TOLERANT = ("uint8_content", "int8_content")


def place16(dev, wire):
    """16 copies of one record, copy s at s bytes past a 256-byte boundary (the payload's source phase walks 0..15)."""
    stride = (len(wire) + 16 + 255) & ~255
    buf = np.zeros(16 * stride + 256, np.uint8)
    rec_off = [s * stride + s for s in range(16)]
    for o in rec_off:
        buf[o: o + len(wire)] = np.frombuffer(wire, np.uint8)
    return dev.upload(buf), rec_off


def two_phase_matrix(dev, wire, cast, out_bytes, pairs):
    """Parse 16 placements of `wire`, then ONE unpack of output 0 of placement s into destination phase d for every (s, d)
    in pairs, each destination in a canary-filled region of its own.  Returns (image, [(s, d, region start, src, dst)])."""
    arena, rec_off = place16(dev, wire)
    n = 16
    off, ln = (C.c_uint64 * n)(*rec_off), (C.c_uint64 * n)(*([len(wire)] * n))
    outs = (N.Output * (4 * n))()
    n_outs, specs, status = (C.c_int32 * n)(), (N.ModelSpec * n)(), (C.c_int32 * n)()
    N.check(dev.lib.b200tfs_parse_responses(dev.ctx, arena, n, off, ln, 4, outs, n_outs, specs, status))
    assert all(status[i] == 0 and n_outs[i] == 1 for i in range(n))
    region = (out_bytes + 64 + 255) & ~255
    base = canary_buffer(dev, region * len(pairs))
    m = len(pairs)
    sel = (N.Output * m)(*[outs[4 * s] for s, _ in pairs])
    dsts = (C.c_void_p * m)(*[base + j * region + 16 + d for j, (_, d) in enumerate(pairs)])
    st = (C.c_int32 * m)()
    N.check(dev.lib.b200tfs_unpack_outputs(dev.ctx, arena, m, sel, (C.c_uint64 * m)(*[rec_off[s] for s, _ in pairs]), dsts,
                                           (C.c_int32 * m)(*([cast or outs[0].dtype] * m)), st))
    assert all(st[j] == 0 for j in range(m))
    o = outs[0]
    first = o.content_off if o.n_runs == 0 else o.runs[0].off
    placed = [(s, d, j * region + 16 + d, arena + rec_off[s] + first, base + j * region + 16 + d) for j, (s, d) in enumerate(pairs)]
    return dev.download(base, region * m), placed, region, o


@pytest.mark.parametrize("case", D1_CASES, ids=[c[0] for c in D1_CASES])
def test_two_phase_unpack_source_by_destination_phase(fresh, case):
    """D1: the full 16 x 16 matrix of source and destination phases at the lengths around the warp / tile, tile, round and
    2- / 3-tile edges (a diagonal of it at 3 tiles and at 3 MiB), every destination inside a canary."""
    name, make, kw, cast, op, ein, eout = case
    dev = fresh()
    vpt = 2048
    full = [(s, d) for s in range(16) for d in range(16)]
    lengths = edge_lengths(16 * vpt, eout) + [(3 << 20) + 16]
    hit, bodies, rounds = set(), set(), set()
    for i, nout in enumerate(lengths):
        nout = nout // eout * eout
        x = make(nout // eout * ein, i)
        wire = wire_oracle.build_predict_response([("x", x)], **kw)
        ref = wire_oracle.decode_predict_response(wire, strict=name not in TOLERANT)["x"]
        want = ref.tobytes() if not cast else wire_oracle.narrow_f32(ref, np.float16 if cast == 19 else ml_dtypes.bfloat16).tobytes()
        assert len(want) == nout
        pairs = full if nout <= 16 * vpt + 17 else [(s, (5 * s + j) % 16) for s in range(16) for j in range(2 if nout < 1 << 20 else 1)]
        image, placed, region, _ = two_phase_matrix(dev, wire, cast, nout, pairs)
        want_img = np.full(image.size, CANARY, np.uint8)
        for s, d, at, src, dst in placed:
            want_img[at: at + nout] = np.frombuffer(want, np.uint8)
            if M.route(nout) == "tile":
                g = M.Geometry(src, dst, nout, op)
                hit.add((g.k, g.dphase))
                bodies.add(g.body())
                rounds.update(r for *_, r in g.tiles(vpt))
        same_image(image, want_img, (name, nout))
    assert hit == {(k, d) for k in range(16) for d in range(16)}, name
    if op in (M.F2H, M.F2B):
        assert bodies >= {"narrow", "narrow0", "narrow1", "narrow2", "narrow3", None} and 2 in rounds
    elif op == M.QUIET_DST:
        assert bodies >= {None, "aligned", "shifted0", "shifted1", "shifted2", "shifted3"}   # head & 3 != 0: the byte generator
    else:
        assert bodies >= {"aligned", "shifted0", "shifted1", "shifted2", "shifted3"}


def _unpacked_rows(x, key):
    """float_val written element by element (tag + 4 bytes each): a gathered source row."""
    dim = b"\x08" + _vi(x.size)
    shape = b"\x12" + _vi(len(dim)) + dim
    body = np.concatenate([np.full((x.size, 1), 0x2D, np.uint8), x.view(np.uint8).reshape(-1, 4)], axis=1).tobytes()
    tp = b"\x08\x01\x12" + _vi(len(shape)) + shape + body
    entry = b"\x0a" + _vi(len(key)) + key + b"\x12" + _vi(len(tp)) + tp
    return b"\x0a" + _vi(len(entry)) + entry


@pytest.mark.parametrize("tile_bytes", [None, 32, 96])
def test_two_phase_unpacked_rows_across_tile_edges(fresh, tile_bytes):
    """D1, gather: rows of unpacked float_val across the tile edges of 32 KB and of 2- and 6-vector tiles, every destination
    phase, against the oracle and inside a canary."""
    dev = fresh(tile_bytes)
    vpt = M.pick_vec_per_tile(132, 1, 32768, override=tile_bytes or 0)
    tiles, dphases = set(), set()
    for i, n in enumerate((513, 8191, 8193, 16385)):
        x = patterns(4 * n, i).view(np.float32)
        wire = _unpacked_rows(x, b"row")
        want = wire_oracle.decode_predict_response(wire)["row"].tobytes()
        assert M.out_bytes(M.QUIET_DST, M.gather(np.frombuffer(wire, np.uint8)[len(wire) - 5 * n + 1:], 4, 5, 4 * n).tobytes()) == want
        pairs = [(s, (3 * s + i) % 16) for s in range(16)]
        image, placed, region, o = two_phase_matrix(dev, wire, 0, 4 * n, pairs)
        runs = [o.runs[q] for q in range(o.n_runs)]
        assert sum(r.count for r in runs) == n and all((r.len, r.stride) == (4, 5) for r in runs)   # rows: the gather
        want_img = np.full(image.size, CANARY, np.uint8)
        for s, d, at, src, dst in placed:
            want_img[at: at + 4 * n] = np.frombuffer(want, np.uint8)
            dphases.add(dst & 15)
        tiles.add(M.tiles_for(4 * n, vpt))
        same_image(image, want_img, (tile_bytes, n))
    assert dphases == set(range(16))
    # every row is tiled (2052 bytes and more): 1..3 tiles of 32 KB, or dozens to thousands of 2- and 6-vector tiles
    assert tiles == {1, 2, 3} if tile_bytes is None else min(tiles) >= 20


# ---- D2 / D3: the single-launch decode, register path and TMA-staged path ---------------------------------------------------
def fused_pair(dev, wire, cast=0, other=None):
    """16 placements of `wire` (source phases 0..15) decoded twice with b200tfs_decode_responses: the first launch walks,
    the second takes the framing template.  other: a record of the same length and other framing, decoded in a third launch
    in place of placement 5 (it misses the template: a staged tile drains its copies, then the record is walked).  Each
    launch into canary-filled slots, compared with the oracle.  Returns [(walked, template, kernel launches)] of the
    launches and (src, dst, wire bytes, n_out, dtype) of every output of the template launch."""
    arena, rec_off = place16(dev, wire)
    n = 16
    wires = [wire] * n
    off, ln = (C.c_uint64 * n)(*rec_off), (C.c_uint64 * n)(*([len(wire)] * n))
    slot = C.c_uint64()
    host = np.frombuffer(wire + b"\0" * 16, np.uint8)
    N.check(dev.lib.b200tfs_decode_slot_bytes(host.ctypes.data, 1, (C.c_uint64 * 1)(0),
                                              (C.c_uint64 * 1)(len(wire)), 0, C.byref(slot), None))
    stride = ((slot.value + 255) & ~255) + 256
    dst = dev.malloc(stride * n)
    N.check(dev.lib.b200tfs_set_decode_cast(dev.ctx, cast))
    deltas, placed = [], []
    for rep in range(3 if other else 2):
        if rep == 2:
            assert len(other) == len(wire) and other != wire
            N.check(dev.lib.b200tfs_memcpy_h2d(dev.ctx, arena + rec_off[5], np.frombuffer(other, np.uint8).ctypes.data, len(other)))
            wires[5] = other
        N.check(dev.lib.b200tfs_memset(dev.ctx, dst, CANARY, stride * n))
        s0, l0 = stats(dev), launches(dev)
        N.check(dev.lib.b200tfs_decode_responses(dev.ctx, arena, n, off, ln, dst, stride))
        outs = (N.Output * (n * N.FUSED_MAX_OUTPUTS))()
        n_outs, status = (C.c_int32 * n)(), (C.c_int32 * n)()
        N.check(dev.lib.b200tfs_decode_results(dev.ctx, n, outs, n_outs, None, status))
        s1 = stats(dev)
        deltas.append((s1[1] - s0[1], s1[0] - s0[0], launches(dev) - l0))
        image = dev.download(dst, stride * n)
        want_img = np.full(image.size, CANARY, np.uint8)
        for r in range(n):
            ref = wire_oracle.decode_predict_response(wires[r])
            assert status[r] == 0 and n_outs[r] == len(ref), (rep, r, status[r])
            for q in range(n_outs[r]):
                o = outs[r * N.FUSED_MAX_OUTPUTS + q]
                key = wires[r][o.key_off: o.key_off + o.key_len].decode()
                v = ref[key]
                if cast and v.dtype == np.float32:
                    v = wire_oracle.narrow_f32(v, np.float16 if cast == 19 else ml_dtypes.bfloat16)
                want = v.tobytes()
                assert o.dst_bytes == len(want), (rep, r, key)
                want_img[r * stride + o.dst_off: r * stride + o.dst_off + len(want)] = np.frombuffer(want, np.uint8)
                narrowed = bool(cast) and ref[key].dtype == np.float32
                at = 0
                for k in range(o.n_runs):
                    run = o.runs[k]
                    nb = run.len // 2 if narrowed else run.len
                    if rep == 1:
                        placed.append((arena + rec_off[r] + run.off, dst + r * stride + o.dst_off + at, run.len, nb, ref[key].dtype))
                    at += nb
        same_image(image, want_img, ("fused", rep))
    return deltas, placed


def launches(dev):
    v = C.c_uint64()
    N.check(dev.lib.b200tfs_kernel_launches(dev.ctx, C.byref(v)))
    return v.value


def stats(dev):
    a, b, c = C.c_uint64(), C.c_uint64(), C.c_uint64()
    N.check(dev.lib.b200tfs_decode_stats(dev.ctx, C.byref(a), C.byref(b), C.byref(c)))
    return a.value + b.value, c.value


def fused_sweep(dev, vpt, lengths, cast=0, cut=True, miss=False, three=False):
    """fused_pair over float32 and float64 payloads of the given byte lengths; a float32 payload is also split in two packed
    occurrences (the second chunk then starts at a destination head that is not 16-byte aligned).  miss: a third launch
    with a same-length record of another key (fused_pair's `other`).  three: the template launch of a narrowing batch runs
    as verify, guarded move and fallback.  Returns the geometries of the template launches."""
    geos = []
    for i, nb in enumerate(lengths):
        cases = [patterns(nb // 4 * 4, i).view(np.float32)]
        if not cast:
            cases.append(patterns(nb // 8 * 8, i + 1).view(np.float64))
        for x in cases:
            key = "k" * (1 + i % 15)
            wires = [wire_oracle.build_predict_response([(key, x)], keep_snan=True)]
            if cut and x.dtype == np.float32 and x.size > 8:
                wires.append(_response_with_chunks(b"c" * (1 + i % 15), x, [x.size // 2 + 1]))
            for w in wires:
                other = wire_oracle.build_predict_response([("j" + key[1:], x)], keep_snan=True) if miss and w is wires[0] else None
                deltas, placed = fused_pair(dev, w, cast, other)
                if three:                                             # verify launch, move_guarded_kernel, fallback launch
                    assert deltas[0][:2] == (16, 0) and deltas[1][2] >= 3, deltas
                else:                                                 # walk, then the template for every placement
                    assert [d[:2] for d in deltas[:2]] == [(16, 0), (0, 16)] and deltas[1][2] == 1, deltas
                if other:
                    assert deltas[2][:2] == (1, 15), deltas           # the record that missed the template was walked
                for src, dst, n_in, n_out, dt in placed:
                    op = M.QUIET_DST if dt == np.float32 else M.COPY
                    if cast and dt == np.float32:
                        geos.append(M.Geometry(src, dst, n_out, M.F2H if cast == 19 else M.F2B))
                    else:
                        geos.append(M.Geometry(src, dst, n_in, op, dec=True))
    return geos


@pytest.mark.parametrize("tile_bytes", [32, 64, 96, 32768])
def test_fused_decode_register_path_at_every_phase(fresh, tile_bytes):
    """D2: decode_fused_kernel, a walking launch then a template launch, source phases 0..15, payloads at tile edges and
    split over two packed occurrences; tiles of 2, 4 and 6 vectors and of 32 KB (the default for small batches)."""
    dev = fresh(tile_bytes)
    vpt = M.pick_vec_per_tile(132, 1, 65536, override=tile_bytes)
    T = 16 * vpt
    lengths = sorted({16, 17 * 4, T + 16, 3 * T + 48, 2 * T - 16, 1000}) if vpt < 16 else [4, 16, T - 16, T + 16, 2 * T + 16, 3 * T + 4]
    geos = fused_sweep(dev, vpt, lengths)
    assert {g.k for g in geos if g.fast and g.nvec} == set(range(16))
    assert any(g.dphase for g in geos)                         # later chunks start at a destination head
    assert any(g.head and g.tail and len(g.tiles(vpt)) >= 2 for g in geos) and any(len(g.tiles(vpt)) >= 3 for g in geos)


STAGED = {32800: (2, 2), 65536: (2, 2048), 98304: (3, 2048), 163840: (5, 2048), 262144: (8, 2048)}


@pytest.mark.parametrize("tile_bytes", sorted(STAGED))
def test_fused_decode_staged_chunks(fresh, tile_bytes):
    """D3: decode_fused_staged_kernel under B200TFS_TILE_BYTES: 2 chunks with a 2-vector second chunk, 2, 3 (refill and
    the wait on parity 1), 5 and 8 chunks; source phases 0..15; lengths ending at chunk edges +- 1 vector and +- 4 bytes;
    and a third launch in which one record of the template's length carries another key: its staged copies are drained
    (staged_drain) before it is walked.

    Not reached, by construction: the staged kernel's move_tile_cold fallback for a QUIET_DST chunk with head & 3 != 0.
    Every output starts 256-byte aligned in its slot and a later chunk starts whole float32 elements further, so a float32
    chunk's head is always a multiple of 4 (the first launch's walk also runs move_tile_cold, but that is the walk, not
    this fallback)."""
    dev = fresh(tile_bytes)
    vpt = M.pick_vec_per_tile(132, 1, 65536, override=tile_bytes)
    assert vpt > M.K_STAGE_VECS
    T, CH = 16 * vpt, 16 * M.K_STAGE_VECS
    edges = sorted({T} | {c * CH for c in range(1, -(-vpt // M.K_STAGE_VECS))})
    lengths = sorted({e + d for e in edges for d in ((-16, -4, 4, 16) if e >= edges[-2] else (-16, 16))} | {T + CH + 16, 2 * T + 4})
    geos = fused_sweep(dev, vpt, lengths, cut=tile_bytes in (32800, 98304), miss=True)
    want_chunks, want_last = STAGED[tile_bytes]
    seen_chunks, lasts, parity1, ks = set(), set(), False, set()
    for g in geos:
        st = g.staged(vpt)
        if st is None:
            continue
        for t, chunks in st:
            if chunks:
                seen_chunks.add(len(chunks))
                lasts.add(chunks[-1][1])
                parity1 |= any(p == 1 for *_, p in chunks)
                ks.add(g.k)
    assert want_chunks in seen_chunks and want_last in lasts, (seen_chunks, lasts)
    assert ks == set(range(16))
    assert parity1 == (want_chunks > 2)


@pytest.mark.parametrize("cast", [19, 14])
def test_fused_decode_staged_narrowing(fresh, cast):
    """D3, casts: the narrowing tile inside decode_fused_staged_cast_kernel at source phases 0..15 and 3-chunk tiles."""
    dev = fresh(98304)
    vpt = M.pick_vec_per_tile(132, 1, 65536, override=98304)
    T = 16 * vpt
    geos = fused_sweep(dev, vpt, [T - 16, T + 4, 2 * T + 4], cast=cast)   # under 4 MiB a batch: one launch, not three
    assert {g.k for g in geos if g.fast} == set(range(16)) and any(r >= 2 for g in geos for *_, r in g.tiles(vpt))


# ---- D5: the three-launch narrowing decode (verify, move_guarded_kernel, fallback) -----------------------------------------
@pytest.mark.parametrize("cast", [19, 14])
def test_three_launch_narrowing_decode(fresh, cast):
    """D5: a narrowing batch of 16 equal-length records (over 4 MiB) whose length the context has seen: the template launch
    runs as verify, move_guarded_kernel over a host-built plan, fallback.  That plan's tiles are 32 KB of output (2048
    vectors: two rounds of body_narrow_q); source phases 0..15 at tile and round edges of the output."""
    dev = fresh()
    vpt = 2048
    T = 16 * vpt
    outs = [8 * T - 16, 8 * T + 2, 8 * T + T // 2 + 16, 9 * T - 2]
    geos = fused_sweep(dev, vpt, [2 * n for n in outs], cast=cast, three=True)
    assert {g.k for g in geos if g.fast} == set(range(16)) and {g.body() for g in geos} >= {"narrow", "narrow1", "narrow3"}
    assert {r for g in geos for *_, r in g.tiles(vpt)} >= {1, 2} and {(g.n_out - g.head) % T for g in geos} >= {T - 16, 2, T // 2 + 16}


# ---- D4: the concatenated decode --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("np_dt", [np.float32, np.float64])
def test_concat_decode_rows_at_every_phase(fresh, np_dt):
    """D4: b200tfs_decode_concat of records whose rows hold 7 elements (28 / 56 bytes), so that the records' values start at
    every element-aligned destination phase, from records placed at every source phase.  Under 64 KB tiles
    (B200TFS_TILE_BYTES=65536: 4096 vectors, two rounds of the same-width bodies) each record crosses tile and round edges.
    Compared with the oracle inside a canary.  (The concatenated decode moves typed fixed-width values only: a 1- or
    2-byte dtype's values are varints there, decoded by the varint kernels, so odd-byte rows do not reach the move engine.)"""
    dev = fresh(65536)
    vpt = 4096
    esz = np.dtype(np_dt).itemsize
    rows = [1, 3, 300] + [80000 // (7 * esz) + 3 * r for r in range(61)]
    arrays = [patterns(7 * k * esz, r).view(np_dt).reshape(k, 7) for r, k in enumerate(rows)]
    wires = [wire_oracle.build_predict_response([("x", a)], keep_snan=True) for a in arrays]
    n = len(wires)
    off, cur = [], 0
    for r, w in enumerate(wires):
        off.append(cur + r % 16)
        cur = (cur + r % 16 + len(w) + 255) & ~255
    buf = np.zeros(cur + 256, np.uint8)
    for o, w in zip(off, wires):
        buf[o: o + len(w)] = np.frombuffer(w, np.uint8)
    coff, cln = (C.c_uint64 * n)(*off), (C.c_uint64 * n)(*[len(w) for w in wires])
    ck = (N.ConcatKey * 1)()
    ck[0].key, ck[0].key_len = b"x", 1
    N.check(dev.lib.b200tfs_concat_layout(buf.ctypes.data, n, coff, cln, 1, ck, 0))
    nb = int(ck[0].bytes)
    refs = [wire_oracle.decode_predict_response(w)["x"] for w in wires]
    want = np.concatenate(refs).tobytes()
    assert nb == len(want), (nb, len(want))
    arena = dev.upload(buf)
    dst = canary_buffer(dev, nb + 512)
    ck[0].dst, ck[0].dst_cap = dst, nb
    N.check(dev.lib.b200tfs_decode_concat(dev.ctx, arena, n, coff, cln, 1, ck))
    res, specs, st = (N.Output * n)(), (N.ModelSpec * n)(), (C.c_int32 * n)()
    N.check(dev.lib.b200tfs_concat_results(dev.ctx, n, 1, res, specs, st))
    assert all(st[r] == N.OK for r in range(n))
    want_img = np.full(nb + 512, CANARY, np.uint8)
    want_img[:nb] = np.frombuffer(want, np.uint8)
    same_image(dev.download(dst, nb + 512), want_img, "concat")
    op = M.QUIET_DST if np_dt is np.float32 else M.COPY
    geos, at = [], 0
    for a, ref, o, w in zip(arrays, refs, off, wires):
        p = w.find(a.tobytes())
        assert p > 0 and w.find(a.tobytes(), p + 1) < 0
        geos.append(M.Geometry(arena + o + p, dst + at, a.nbytes, op))
        at += a.nbytes
    big = [g for g in geos if g.n_out > 16 * vpt]
    assert {g.dphase for g in big} == set(range(0, 16, 4 if esz == 4 else 8)) and {g.k for g in big} == set(range(16))
    assert {g.body() for g in big} >= {"aligned", "shifted0", "shifted1", "shifted2", "shifted3"}
    assert any(len(g.tiles(vpt)) >= 2 and g.tiles(vpt)[0][3] == 2 for g in big)
