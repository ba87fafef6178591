"""The string-column routes at their edges, through the C ABI, byte for byte against tests/strcol_ref.py: the padded DT_STRING request
encode, the concatenated and padded DT_STRING response decodes, and the tf.Example bytes_list encode.  Every destination is filled
with a canary and has slack behind it; bytes outside the promised ranges must keep it.  Each case asks the geometry model whether it
reached the edge it is named for, so a retuned constant moves the case instead of letting it pass without reaching anything."""
import ctypes as C

import numpy as np
import pytest

import example_ref as E
import golden_util as G
import strcol_ref as S
import string_responses as SR
from devutil import Dev
from min_tfs_client import _native as N
from min_tfs_client.codec import BytesColumn, RaggedColumn

pytestmark = pytest.mark.gpu

CANARY = 0xC5
SLACK = 1 << 16
EDGE_LENS = [0, 1, 15, 16, 17, 63, 64, 65, 127, 128, 16383, 16384, 16385, (1 << 21) - 1, 1 << 21]
SHORT_LENS = [0, 1, 15, 16, 17, 63, 64, 65, 127, 128]


def distinct(lens, seed=0):
    """one string per length, NUL and high bytes included"""
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, int(n), dtype=np.uint8).tobytes() for n in lens]


@pytest.fixture
def dev():
    d = Dev()
    yield d
    d.close()


def canvas(dev, nbytes):
    """(base of the usable range, allocation start) of a canary-filled device buffer with SLACK on both sides, 256-aligned"""
    total = nbytes + 2 * SLACK + 256
    p0 = dev.malloc(total)
    fill = np.full(total, CANARY, np.uint8)
    N.check(dev.lib.b200tfs_memcpy_h2d(dev.ctx, p0, fill.ctypes.data, total))
    dev.sync()
    return (p0 + SLACK + 255) & ~255, p0, total


def same(got, want, what):
    """got == want (byte strings or int arrays), reporting the first difference instead of a diff of the whole thing"""
    g = np.frombuffer(got, np.uint8) if isinstance(got, bytes) else np.asarray(got)
    w = np.frombuffer(want, np.uint8) if isinstance(want, bytes) else np.asarray(want)
    if len(g) != len(w) or not np.array_equal(g, w):
        d = np.flatnonzero(g[: min(len(g), len(w))] != w[: min(len(g), len(w))])
        raise AssertionError((what, len(g), len(w), int(d[0]) if len(d) else None))


def untouched(mem, allowed):
    """every byte outside the allowed [a, b) ranges still holds the canary"""
    inside = np.zeros(len(mem), bool)
    for a, b in allowed:
        inside[a:b] = True
    bad = np.flatnonzero((mem != CANARY) & ~inside)
    assert not len(bad), bad[:8]


# ---- padded encode ---------------------------------------------------------------------------------------------------------
def column(dist, pattern, start=0):
    """(data, offsets) of the column of strings dist[pattern[i]], `start` bytes of junk in front, a few behind"""
    lens = S.lens_of(dist)[np.asarray(pattern, np.int64)]
    sz = np.r_[0, np.cumsum(S.lens_of(dist))]
    flat = S.flat_of(dist)
    off = np.zeros(len(lens) + 1, np.int64)
    np.cumsum(lens, out=off[1:])
    idx = np.repeat(sz[:-1][pattern] - off[:-1], lens) + np.arange(int(off[-1])) if len(lens) else np.zeros(0, np.int64)
    data = np.concatenate([np.full(start, 0x5A, np.uint8), flat[idx], np.full(16, 0x5B, np.uint8)])
    return data, off + start


def encode_ref(dist, pattern, dims, shapes):
    """every request's wire: request r's box of the column (strings dist[pattern]) as its DT_STRING input "s" """
    shapes = np.asarray(shapes, np.int64).reshape(len(shapes), -1)
    r0 = np.r_[0, np.cumsum(shapes[:, 0])]
    out, jobs = [], []
    for r in range(len(shapes)):
        idx, bd = S.box_index(dims, int(r0[r]), shapes[r])
        p = np.asarray(pattern, np.int64)[idx]
        body = S.tiled_values(dist, p, 0x42)[1].tobytes()
        out.append(S.predict_request("m", 3, {"s": S.tensor_proto(body, bd)}))
        jobs.append(S.EncodeJob(S.lens_of(dist)[p], idx))
    return out, jobs


def run_encode(dev, dist, pattern, dims, shapes, start=0, bad_at=None):
    """encode through b200tfs_encode_padded_requests_columns_async; bad_at = (request, string): that string's end drops below its
    start.  Returns (rec_off, rec_len, status of the call, the arena image, the arena's offset in it)"""
    data, off = column(dist, pattern, start)
    if bad_at is not None:
        shapes2 = np.asarray(shapes, np.int64).reshape(len(shapes), -1)
        first = int(np.r_[0, np.cumsum(shapes2[:, 0])][bad_at[0]]) * int(np.prod(dims[1:], dtype=np.int64))
        off = off.copy()
        off[first + bad_at[1] + 1] = off[first + bad_at[1]] - 1
    S2 = np.ascontiguousarray(np.asarray(shapes, np.int64))
    n, cols = len(S2), (S2.shape[1] if S2.ndim == 2 else 1)
    dd = dev.upload(np.concatenate([data, np.zeros(SLACK, np.uint8)]))
    do, ds = dev.upload(off), dev.upload(S2)
    d = (C.c_int64 * len(dims))(*dims)
    ts = (N.Tensor * 1)(N.Tensor(data=dd, src_dtype=7, wire_dtype=7, rank=len(dims), flags=N.F_DEVICE_DATA, dims=d, key=b"s",
                                 key_len=1, packed_len=0))
    pins = (N.PadInput * 1)(N.PadInput(shapes=ds, cols=cols))
    bs = (N.Bytes * 1)(N.Bytes(offsets=do, data_len=len(data), flags=N.F_DEVICE_DATA))
    req = N.Request(model_name=b"m", model_name_len=1, has_version=1, order=N.ORDER_UPB, version=3, n_inputs=1, flags=0, inputs=ts)
    cap = C.c_uint64()
    N.check(dev.lib.b200tfs_padded_request_columns_arena_size(n, C.byref(req), bs, C.byref(cap)))
    arena, p0, total = canvas(dev, cap.value)
    N.check(dev.lib.b200tfs_encode_padded_requests_columns_async(dev.ctx, n, C.byref(req), pins, bs, arena, cap.value))
    ro, rl = (C.c_uint64 * n)(), (C.c_uint64 * n)()
    rc = dev.lib.b200tfs_encode_results(dev.ctx, n, ro, rl)
    return list(ro), list(rl), rc, dev.download(p0, total), arena - p0


def check_encode(dev, dist, pattern, dims, shapes, start=0, bad_at=None):
    ref, jobs = encode_ref(dist, pattern, dims, shapes)
    ro, rl, rc, mem, a0 = run_encode(dev, dist, pattern, dims, shapes, start, bad_at)
    allowed = []
    for r, w in enumerate(ref):
        if bad_at is not None and r == bad_at[0]:
            assert rl[r] == 0, r
            continue
        same(mem[a0 + ro[r]: a0 + ro[r] + rl[r]].tobytes(), w, r)
        allowed.append((a0 + ro[r], a0 + ro[r] + rl[r]))
    assert rc == (N.E_SHAPE if bad_at is not None else N.OK)
    untouched(mem, allowed)
    return ref, jobs, ro


@pytest.mark.parametrize("m", [255, 256, 257, 65535, 65536, 65537, 131073])
def test_encode_tiles_and_counter_groups(dev, m):
    """one job of m strings between two others, so the big job's tiles start mid-group in the shared tables and it reaches one,
    two or three counter groups"""
    dist = distinct(SHORT_LENS, 1)
    rng = np.random.default_rng(m)
    rows = np.array([300, m, 77], np.int64)
    pattern = rng.integers(0, len(dist), int(rows.sum()))
    _, jobs, _ = check_encode(dev, dist, pattern, (int(rows.sum()),), rows, start=3)
    big = jobs[1]
    assert big.tiles == -(-m // S.K_VAR_THREADS)
    assert big.groups == -(-big.tiles // S.K_GROUP_TILES)
    assert jobs[0].tiles % S.K_GROUP_TILES                  # the big job's first tile is not a group's first
    if m > S.K_VAR_THREADS * S.K_GROUP_TILES:
        assert big.groups >= 2 and (big.group_of_tile > 0).any()


@pytest.mark.parametrize("n_cta", [0, 1, 2, 256])
def test_encode_cta_tier_beside_lane_and_warp_tiers(dev, n_cta):
    """tiles holding n_cta strings over kUnpadStrBlockCopy bytes; the 256 case fills long_*, the others sit next to lane- and
    warp-tier strings in the same warps"""
    lens = [0, 1, 64, 65, 200, S.K_BLOCK, S.K_BLOCK + 1, (1 << 21) - 1]
    dist = distinct(lens, 2)
    per = S.K_VAR_THREADS
    rng = np.random.default_rng(n_cta)
    tile = rng.integers(0, 5, per)
    tile[rng.choice(per, n_cta, replace=False)] = rng.choice([6, 7, 6, 6], n_cta) if n_cta < per else 6
    pattern = np.concatenate([rng.integers(0, 5, 37), tile, rng.integers(0, 6, 90)])
    rows = np.array([37, per, 90], np.int64)
    _, jobs, _ = check_encode(dev, dist, pattern, (len(pattern),), rows)
    assert jobs[1].cta_per_tile.tolist() == [n_cta]
    if 0 < n_cta < per:
        tiers = {t for _, ts in S.warp_rounds(jobs[1].lens, cta=True) for t in ts}
        assert tiers == {"lane", "warp", "cta"}


MIXES = {"all_lane": [False] * 32, "all_warp": [True] * 32, "only_lane0": [True] + [False] * 31,
         "only_lane31": [False] * 31 + [True], "alternating": [i % 2 == 1 for i in range(32)]}


@pytest.mark.parametrize("start", range(16))
def test_encode_lane_mixes_at_every_phase(dev, start):
    """warps of every lane mix, warp-tier strings of different lengths in one warp; source phase `start` (offsets[0]) and every
    destination phase through the bytes in front"""
    lens = [0, 1, 15, 16, 17, 63, 64, 65, 127, 128, 300, 4000]
    dist = distinct(lens, 3)
    rng = np.random.default_rng(100 + start)
    reqs, leads = [], []
    for lead in range(16):                                      # `lead` one-byte strings in front shift the rest by 3 bytes each
        for name, long in MIXES.items():
            w = np.where(long, rng.choice([7, 8, 9, 10, 11], 32), rng.integers(0, 7, 32))
            reqs.append(np.r_[np.ones(lead, np.int64), w])
            leads.append(lead)
    rows = np.array([len(p) for p in reqs], np.int64)
    pattern = np.concatenate(reqs)
    ref, jobs, ro = check_encode(dev, dist, pattern, (len(pattern),), rows, start=start)
    mixes, src, dst = set(), set(), set()
    data_off = np.r_[0, np.cumsum(S.lens_of(dist)[pattern])] + start
    first = np.r_[0, np.cumsum(rows)]
    for r, job in enumerate(jobs):
        # where request r's string bytes land: its string_val body is the end of the record
        sz = S.tiled_values(dist, pattern[first[r]: first[r + 1]], 0x42)[0]
        body0 = len(ref[r]) - int(sz.sum())
        at = ro[r] + body0 + np.cumsum(sz) - sz + 1 + E.vlen(job.lens)
        long = job.lens > S.K_LANE
        src |= S.phases(data_off[first[r]: first[r + 1]][long])
        dst |= S.phases(at[long])
        mixes |= {S.lane_mix(mask) for mask, _ in S.warp_rounds(job.lens)}     # the kernel's warps start at the job's first string
    assert {"all_lane", "all_warp", "only_lane0", "only_lane31", "alternating"} <= mixes
    assert dst == set(range(16)) and len(src) > 1


def test_encode_trimmed_rank3_boxes_cross_rows(dev):
    dist = distinct(SHORT_LENS + [300], 4)
    rng = np.random.default_rng(5)
    dims = (120, 9, 40)
    n = 12
    Sh = np.stack([np.full(n, 10), rng.integers(5, 10, n), rng.integers(1, 40, n)], 1).astype(np.int64)
    Sh[3] = [10, 9, 40]                                         # one full box: one stretch
    pattern = rng.integers(0, len(dist), int(np.prod(dims)))
    _, jobs, _ = check_encode(dev, dist, pattern, dims, Sh, start=9)
    assert sum(len(j.crossing_tiles) for j in jobs) > n
    assert not jobs[3].crossing_tiles


def test_encode_broadcast_string_read_by_every_request(codec):
    dist = distinct(EDGE_LENS[:13], 6)
    x = np.arange(40, dtype=np.float32).reshape(20, 2)
    rows = np.array([3, 0, 7, 10], np.int64)
    bdata, boff = column(dist, np.arange(len(dist)), start=5)
    got = codec.encode_predict_requests_padded("m", {"x": x}, {"x": rows}, broadcast={"b": BytesColumn(bdata, boff, (len(dist),))},
                                               model_version=3)
    tp_b = S.tensor_proto(S.string_val_body(dist), (len(dist),))
    r0 = np.r_[0, np.cumsum(rows)]
    import padded_strings_ref as PS
    for r in range(len(rows)):
        tx = PS.numeric_proto(x[r0[r]: r0[r + 1]]).SerializeToString()
        assert got[r] == S.predict_request("m", 3, {"x": tx, "b": tp_b}), r


@pytest.mark.parametrize("at", [255, 256])
def test_encode_offsets_violation_at_a_tile_edge(dev, at):
    dist = distinct(SHORT_LENS, 7)
    rng = np.random.default_rng(at)
    rows = np.array([100, 600, 50], np.int64)
    pattern = rng.integers(1, len(dist), int(rows.sum()))       # no empty strings: the decrease always breaks the rule
    check_encode(dev, dist, pattern, (int(rows.sum()),), rows, bad_at=(1, at))


def test_encode_every_edge_length(dev):
    dist = distinct(EDGE_LENS, 8)
    pattern = np.r_[np.arange(len(dist)), np.arange(len(dist))[::-1]]
    rows = np.array([len(dist), len(dist)], np.int64)
    _, jobs, _ = check_encode(dev, dist, pattern, (len(pattern),), rows, start=11)
    assert {t for j in jobs for _, ts in S.warp_rounds(j.lens, cta=True) for t in ts} == {"lane", "warp", "cta"}


# ---- response decodes: records placed at chosen addresses ------------------------------------------------------------------------
def place(recs, skews):
    """host arena with record i at an offset whose skew mod 128 is skews[i]; (buf, rec_off, rec_len)"""
    off, cur = [], 0
    for w, s in zip(recs, skews):
        cur = ((cur + S.LINE - 1) // S.LINE) * S.LINE + int(s)
        off.append(cur)
        cur += len(w)
    buf = np.zeros(cur + 256, np.uint8)
    for w, o in zip(recs, off):
        buf[o: o + len(w)] = np.frombuffer(w, np.uint8)
    return buf, (C.c_uint64 * len(recs))(*off), (C.c_uint64 * len(recs))(*[len(w) for w in recs])


def str_resp(*pairs):
    """a PredictResponse of (key, strings, dims) string outputs and a model_spec"""
    return SR.response(*[(k, SR.string_tensor(s, list(d))) for k, s, d in pairs])


def run_concat(dev, recs, keys, skews=None, data_caps=None, offset_caps=None):
    n, nk = len(recs), len(keys)
    buf, off, ln = place(recs, skews if skews is not None else [0] * n)
    ck, sc = (N.ConcatKey * nk)(), (N.ConcatStrings * nk)()
    kb = [k.encode() for k in keys]
    for i, k in enumerate(kb):
        ck[i].key, ck[i].key_len = k, len(k)
    N.check(dev.lib.b200tfs_concat_strings_layout(buf.ctypes.data, n, off, ln, nk, ck, sc, 0))
    arena = dev.upload(buf)
    bufs = []
    for i in range(nk):
        oc = int(ck[i].bytes) if offset_caps is None else offset_caps[i]
        dc = int(sc[i].data_bytes) if data_caps is None else data_caps[i]
        o, o0, ot = canvas(dev, oc)
        d, d0, dt = canvas(dev, dc)
        ck[i].dst, ck[i].dst_cap, sc[i].data, sc[i].data_cap = o, oc, d, dc
        bufs.append((o - o0, o0, ot, d - d0, d0, dt, oc, dc))
    N.check(dev.lib.b200tfs_decode_concat_strings(dev.ctx, arena, n, off, ln, nk, ck, sc))
    outs = (N.Output * (n * nk))()
    N.check(dev.lib.b200tfs_concat_results(dev.ctx, n, nk, outs, None, None))
    mem = [(dev.download(b[1], b[2]), dev.download(b[4], b[5])) for b in bufs]
    return outs, bufs, mem, (off, ln)


def check_concat(dev, parts, keys, skews=None, data_caps=None, recs=None, noncanonical=()):
    """parts[k][r]: record r's strings of key k; recs: the records when they are not plain responses of those; noncanonical:
    (record, key) pairs whose strings the device walk must refuse.  Checks every OK pair's offsets and bytes, offsets[m] behind the
    last OK pair, statuses against the scan model and the canaries."""
    n, nk = len(parts[0]), len(keys)
    if recs is None:
        recs = [str_resp(*[(keys[k], parts[k][r], (len(parts[k][r]),)) for k in range(nk)]) for r in range(n)]
    offset_caps = [8 * (sum(len(p) for p in parts[k]) + 1) for k in range(nk)]
    outs, bufs, mem, _ = run_concat(dev, recs, keys, skews, data_caps, offset_caps)
    models = []
    for k in range(nk):
        a0, _, _, d0, _, _, oc, dc = bufs[k]
        om, dm = mem[k]
        ok = [(r, k) not in noncanonical for r in range(n)]
        st, first, last = S.concat_scan([S.lens_of(parts[k][r]).sum() for r in range(n)], ok, dc)
        models.append((st, first, last))
        allowed_o, allowed_d = [(a0, a0 + oc)], []
        for r in range(n):
            o = outs[r * nk + k]
            want = {"ok": N.OK, "size": N.E_SIZE, "skip": N.E_NONCANONICAL}[st[r]]
            assert o.status == want, (k, r, o.status, st[r])
            if st[r] != "ok":
                continue
            m = len(parts[k][r])
            got = om[a0 + o.dst_off: a0 + o.dst_off + 8 * m].view(np.int64)
            same(got, (first[r] + np.r_[0, np.cumsum(S.lens_of(parts[k][r]))[:-1]])[:m], (k, r))
            same(dm[d0 + first[r]: d0 + first[r] + len(b"".join(parts[k][r]))].tobytes(), b"".join(parts[k][r]), (k, r))
            allowed_d.append((d0 + first[r], d0 + first[r] + len(b"".join(parts[k][r]))))
        if last is not None:
            lr = max(r for r in range(n) if st[r] == "ok")
            o = outs[lr * nk + k]
            assert om[a0 + o.dst_off + 8 * len(parts[k][lr]): a0 + o.dst_off + 8 * len(parts[k][lr]) + 8].view(np.int64)[0] == last
        untouched(om, allowed_o)
        untouched(dm, allowed_d)
    return outs, models, recs


CHUNK_COUNTS = [255, 256, 257, 0, 1, 513, 0, 0, 256, 31, 32, 33]


@pytest.mark.parametrize("nk", [1, 3, 8])
def test_concat_chunk_edges_and_ties(dev, nk):
    """pairs of 255/256/257 strings and zero-string pairs between them, over up to B200TFS_CONCAT_MAX_KEYS string keys: chunk0
    ties the binary search must step over"""
    dist = distinct(SHORT_LENS + [300], 9)
    rng = np.random.default_rng(nk)
    keys = ["k%d" % k for k in range(nk)]
    n = len(CHUNK_COUNTS)
    parts = [[[dist[i] for i in rng.integers(0, len(dist), CHUNK_COUNTS[(r + k) % n])] for r in range(n)] for k in range(nk)]
    _, models, recs = check_concat(dev, parts, keys, skews=[(17 * r + 5) % S.LINE for r in range(n)])
    # the copy's warp-tier strings: every destination phase (data is 256-aligned) and every lane mix of the kernel's rounds
    dst, mixes = set(), set()
    for k in range(nk):
        for r in range(n):
            lens = S.lens_of(parts[k][r])
            at = models[k][1][r] + np.cumsum(lens) - lens
            dst |= S.phases(at[lens > S.K_LANE])
            mixes |= {S.lane_mix(mask) for mask, _ in S.warp_rounds(lens)}
    assert dst == set(range(16)) and {"all_lane", "mixed"} <= mixes
    ch, c0, total = S.concat_chunks([[len(parts[k][r]) for r in range(n)] for k in range(nk)], np.ones((nk, n), bool))
    assert S.tied_pairs(ch, c0)
    owners = [S.pair_of(c0, c) for c in range(total)]
    assert all(ch[q] for q in owners) and sorted(set(owners)) == [q for q in range(len(ch)) if ch[q]]
    assert {255, 256, 257} <= {len(p) for ps in parts for p in ps}


def test_concat_bad_pairs_between_good_ones(dev):
    """pairs that hold strings but get no chunks, between good pairs at chunk edges: E_SIZE pairs at the end of key k0 (not the
    last key, so they tie with k1's first pairs), and an E_NONCANONICAL pair of k1 (its TensorProto split over two `value`
    occurrences) between good ones; zero-string pairs beside them"""
    dist = distinct(SHORT_LENS, 10)
    rng = np.random.default_rng(11)
    counts = [256, 0, 257, 0, 255, 256, 1]
    n, keys = len(counts), ["k0", "k1", "k2"]
    parts = [[[dist[i] for i in rng.integers(1, len(dist), counts[(r + k) % n])] for r in range(n)] for k in range(3)]
    assert len(parts[1][3]) > 100 and parts[1][4]
    recs = []
    for r in range(n):
        entries = [(keys[k], SR.string_tensor(parts[k][r], [len(parts[k][r])])) for k in range(3)]
        rec = b"".join(G.entry(k, tp) for k, tp in entries)
        if r == 3:
            s = parts[1][3]
            split = G.ld(0x0A, G.ld(0x0A, b"k1") + G.ld(0x12, SR.string_tensor(s[:100], [len(s)])) + G.ld(0x12, SR.strings_body(s[100:])))
            rec = G.entry("k0", entries[0][1]) + split + G.entry("k2", entries[2][1])
        recs.append(rec + G.mspec())
    nbytes = [sum(len(b"".join(parts[k][r])) for r in range(n)) for k in range(3)]
    cap0 = sum(len(b"".join(parts[0][r])) for r in range(n - 2))          # k0: the last two pairs do not fit
    outs, models, _ = check_concat(dev, parts, keys, skews=[0, 64, 127, 1, 96, 33, 5], data_caps=[cap0] + nbytes[1:], recs=recs,
                                   noncanonical={(3, 1)})
    assert models[0][0][-2:] == ["size", "size"] and models[1][0][3] == "skip" and "size" not in models[1][0] + models[2][0]
    ok = [[st == "ok" for st in m[0]] for m in models]
    ch, c0, total = S.concat_chunks([[len(parts[k][r]) for r in range(n)] for k in range(3)], ok)
    tied = S.tied_pairs(ch, c0)
    assert {n - 2, n - 1, n + 3} <= set(tied)                   # (k0, r5), (k0, r6) and (k1, r3): strings, no chunks, a tie


@pytest.mark.parametrize("cut", ["exact", "short"])
def test_concat_data_cap_cuts_at_a_pair(dev, cut):
    """data_cap ends exactly behind pair r, or one byte short of it: a pair's bytes count in the running position whether or not
    they fit, so every pair behind the first E_SIZE pair of the key - zero-byte ones too - is E_SIZE, and offsets[m] stands behind
    the last OK pair"""
    dist = distinct([3, 70, 1, 0], 12)
    per = [[0, 1, 2], [1, 1], [], [3, 3], [0], [2, 1, 0]]
    parts = [[[dist[i] for i in p] for p in per]]
    r = 1
    cap = sum(len(b"".join(parts[0][q])) for q in range(r + 1)) - (cut == "short")
    outs, models, _ = check_concat(dev, parts, ["s"], skews=[3, 9, 27, 81, 115, 0], data_caps=[cap])
    # exact: the zero-byte pairs 2 and 3 start at data_cap and fit; short: they start past it, behind pair 1's bytes
    assert models[0][0] == (["ok"] * 4 + ["size"] * 2 if cut == "exact" else ["ok"] + ["size"] * 5)


def test_concat_copy_warps_stride(dev):
    """more chunks than the copy grid has warps (from the grid formula and this device's SM count)"""
    import torch
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    dist = distinct([0, 5, 64, 65], 13)
    n = sm * 64 + 300
    rng = np.random.default_rng(14)
    pick = rng.integers(0, len(dist), n)
    parts = [[[dist[i]] for i in pick]]
    recs = [str_resp(("s", p, (1,))) for p in parts[0]]
    check_concat(dev, parts, ["s"], recs=recs, skews=[(7 * r) % S.LINE for r in range(n)])
    grid = S.concat_copy_grid([len(w) for w in recs], 1, sm)
    assert S.copy_strides(n, grid)


def skew_records(seed):
    """records whose strings put tags and length varints across line edges, and a long string whose skip leaves both cached lines"""
    rng = np.random.default_rng(seed)
    out = []
    for s in range(S.LINE):
        lens = [int(x) for x in rng.choice([0, 1, 126, 127, 128, 129, 200], 14)] + [900, 5, 130, 1]
        out.append([bytes([(s + i) & 0xFF]) * L for i, L in enumerate(lens)])
    return out


def walk_model(recs, buf_off, key_parts):
    """(records with a tag/varint across a line edge, records with a cold jump) from where each string field really lies"""
    cross = jumps = 0
    for w, a, strs in zip(recs, buf_off, key_parts):
        body = SR.strings_body(strs)
        b0 = w.find(body)
        assert b0 > 0 and w.find(body, b0 + 1) < 0
        f = S.string_fields(b0, S.lens_of(strs))
        cross += bool(S.crossing_varints(S.walk_lines(a, f)))
        jumps += S.cold_jumps(a, len(w), f) > 0
    return cross, jumps


def test_concat_index_walk_at_every_skew(dev):
    strs = skew_records(15)
    recs = [str_resp(("s", p, (len(p),))) for p in strs]
    skews = list(range(S.LINE))
    check_concat(dev, [strs], ["s"], skews=skews, recs=recs)
    _, off, _ = place(recs, skews)
    cross, jumps = walk_model(recs, list(off), strs)
    assert cross > 8 and jumps == S.LINE


# ---- padded decode ---------------------------------------------------------------------------------------------------------
def run_padded(dev, recs, keys, tails, pads, skews=None, data_caps=None):
    n, nk = len(recs), len(keys)
    buf, off, ln = place(recs, skews if skews is not None else [0] * n)
    pk, ps = (N.PadKey * nk)(), (N.PaddedStrings * nk)()
    kb = [k.encode() for k in keys]
    for i, k in enumerate(kb):
        pk[i].key, pk[i].key_len = k, len(k)
    N.check(dev.lib.b200tfs_padded_strings_layout(buf.ctypes.data, n, off, ln, nk, pk, ps, 0))
    arena = dev.upload(buf)
    bufs = []
    for i in range(nk):
        m = int(pk[i].dims[0]) * int(np.prod(tails[i], dtype=np.int64))
        oc = 8 * (m + 1)
        dc = int(ps[i].data_bytes) + (m - int(ps[i].strings)) * len(pads[i]) if data_caps is None else data_caps[i]
        o, o0, ot = canvas(dev, oc)
        d, d0, dt = canvas(dev, dc)
        pk[i].dst, pk[i].dst_cap, pk[i].rank = o, oc, len(tails[i]) + 1
        for d_, x in enumerate(tails[i]):
            pk[i].dims[d_ + 1] = x
        ps[i].data, ps[i].data_cap, ps[i].pad, ps[i].pad_len = d, dc, C.cast(C.c_char_p(pads[i]), C.c_void_p), len(pads[i])
        bufs.append((o - o0, o0, ot, d - d0, d0, dt, oc, dc))
    N.check(dev.lib.b200tfs_decode_padded_strings(dev.ctx, arena, n, off, ln, nk, pk, ps))
    outs = (N.Output * (n * nk))()
    N.check(dev.lib.b200tfs_padded_results(dev.ctx, n, nk, outs, None, None))
    mem = [(dev.download(b[1], b[2]), dev.download(b[4], b[5])) for b in bufs]
    return outs, bufs, mem


def check_padded(dev, keys, parts, tails, pads, skews=None, data_caps=None):
    """parts[k][r] = (strings, dims) of record r's output for key k"""
    n, nk = len(parts[0]), len(keys)
    recs = [str_resp(*[(keys[k],) + tuple(parts[k][r]) for k in range(nk)]) for r in range(n)]
    outs, bufs, mem = run_padded(dev, recs, keys, tails, pads, skews, data_caps)
    cuts = []
    for k in range(nk):
        a0, _, _, d0, _, _, oc, dc = bufs[k]
        om, dm = mem[k]
        re = int(np.prod(tails[k], dtype=np.int64))
        # the scan: each record's bytes, own and pads; the rows in use end at the first record past data_cap
        at, cut, st = 0, None, []
        for r in range(n):
            strs = S.padded_strings([parts[k][r]], tails[k], pads[k])
            b = sum(len(x) for x in strs)
            st.append(N.E_SIZE if strs and at + b > dc else N.OK)
            if st[-1] == N.E_SIZE and cut is None:
                cut = (r, at)
            at += b
        used = n if cut is None else cut[0]
        data, offs = S.padded_column([parts[k][r] for r in range(used)], tails[k], pads[k])
        m = len(offs) - 1
        assert [outs[r * nk + k].status for r in range(n)] == st, k
        same(om[a0: a0 + 8 * (m + 1)].view(np.int64), offs, k)
        same(dm[d0: d0 + len(data)].tobytes(), data.tobytes(), k)
        rows_before = sum(p[1][0] for p in parts[k][:used])
        assert m == rows_before * re
        untouched(om, [(a0, a0 + max(oc, 8 * (m + 1)))])           # entries of a record cut for its bytes may hold scratch
        untouched(dm, [(d0, d0 + len(data))])
        cuts.append(cut)
    return recs, cuts


@pytest.mark.parametrize("pad_len", [0, 1, 64, 65, 16385])
def test_padded_pad_lengths_across_records_and_keys(dev, pad_len):
    dist = distinct(SHORT_LENS + [300, 16385], 16)
    rng = np.random.default_rng(pad_len)
    pad = bytes(rng.integers(0, 256, pad_len, dtype=np.uint8))
    n = 9
    parts = []
    for k in range(2):
        pk = []
        for r in range(n):
            dims = (int(rng.integers(0, 3)), int(rng.integers(0, 7)) if r % 4 else 0)      # records of no own strings too
            m = dims[0] * dims[1]
            pk.append(([dist[i] for i in rng.integers(0, len(dist), m)], dims))
        parts.append(pk)
    tails = [(max(p[1][1] for p in parts[k]) + k,) for k in range(2)]
    check_padded(dev, ["a", "b"], parts, tails, [pad, pad], skews=[(31 * r) % S.LINE for r in range(n)])
    pos = S.padded_positions([(parts[k], tails[k], pad) for k in range(2)])
    rec_rounds, key_rounds = S.padded_rounds(pos)
    assert rec_rounds and key_rounds
    assert any(not own for _, _, own, _ in pos) and {S.tier(pad_len)} <= {S.tier(L) for _, _, own, L in pos if not own}


@pytest.mark.parametrize("rank", [2, 3, 4])
def test_padded_ranks_last_axis_one_and_full(dev, rank):
    dist = distinct(SHORT_LENS, 17)
    rng = np.random.default_rng(rank)
    n, D = 7, 5
    parts = []
    for r in range(n):
        dims = (int(rng.integers(1, 3)),) + tuple(int(rng.integers(1, D + 1)) for _ in range(rank - 2)) + ((1, D)[r % 2],)
        parts.append(([dist[i] for i in rng.integers(0, len(dist), int(np.prod(dims)))], dims))
    tail = tuple(max(p[1][d] for p in parts) for d in range(1, rank))
    check_padded(dev, ["s"], [parts], [tail], [b"<>"])
    assert sum(S.place_carries(p[1]) for p in parts) > 0
    assert {p[1][-1] for p in parts} == {1, D}


@pytest.mark.parametrize("cut", ["exact", "short"])
def test_padded_data_cap_cuts_rows(dev, cut):
    dist = distinct([3, 70, 1, 0], 18)
    per = [(2, 2), (1, 3), (0, 3), (2, 1), (1, 2)]
    rng = np.random.default_rng(19)
    parts = [([dist[i] for i in rng.integers(0, 4, a * b)], (a, b)) for a, b in per]
    tail = (3,)
    pad = b"PAD"
    r = 1
    cap = sum(sum(len(x) for x in S.padded_strings([parts[q]], tail, pad)) for q in range(r + 1)) - (cut == "short")
    _, cuts = check_padded(dev, ["s"], [parts], [tail], [pad], data_caps=[cap])
    assert cuts[0][0] == (r + 2 if cut == "exact" else r)       # record 2 has no rows: the cut passes over it


def test_padded_index_walk_at_every_skew(dev):
    strs = skew_records(20)
    parts = [(p, (1, len(p))) for p in strs]
    skews = list(range(S.LINE))
    recs, _ = check_padded(dev, ["s"], [parts], [(max(len(p) for p in strs),)], [b"~"], skews=skews)
    _, off, _ = place(recs, skews)
    cross, jumps = walk_model(recs, list(off), strs)
    assert cross > 8 and jumps == S.LINE


def test_padded_two_keys_last_key_positions(dev):
    """the copy's key search over several keys: positions of the last key must find it"""
    dist = distinct(SHORT_LENS, 21)
    rng = np.random.default_rng(22)
    n = 5
    parts = [[([dist[i] for i in rng.integers(0, len(dist), 2 * t)], (2, t)) for t in rng.integers(0, 4, n).tolist()] for _ in range(3)]
    tails = [(3,), (4,), (5,)]
    check_padded(dev, ["a", "b", "c"], parts, tails, [b"x", b"", b"yz"])


# ---- tf.Example bytes rows -------------------------------------------------------------------------------------------------------
def bytes_column(strs, shape, start=0):
    lens = S.lens_of(strs)
    off = np.r_[0, np.cumsum(lens)].astype(np.int64) + start
    return BytesColumn(np.concatenate([np.full(start, 0xEE, np.uint8), S.flat_of(strs), np.full(3, 0xEE, np.uint8)]), off, shape)


ROUNDS = [0, 31, 32, 33, 64, 65]


@pytest.mark.parametrize("target", [None, "examples"], ids=["classify", "predict"])
def test_example_bytes_rows_in_32_string_rounds(codec, target):
    dist = distinct(SHORT_LENS + [300], 23)
    rng = np.random.default_rng(24)
    n, L = len(ROUNDS), max(ROUNDS)
    plain = {w: bytes_column([dist[i] for i in rng.integers(0, len(dist), n * w)], (n, w), start=w % 16) for w in ROUNDS[1:]}
    rag = bytes_column([dist[i] for i in rng.integers(0, len(dist), n * L)], (n, L), start=7)
    d = {"p%02d" % w: c for w, c in plain.items()}
    d["r"] = RaggedColumn(rag, np.array(ROUNDS, np.int64))
    d["x"] = np.arange(n, dtype=np.float32)
    kw = {} if target is None else {"predict_input": target}
    got = codec.encode_example_requests([("m", 1, d)], **kw)[0]
    assert got == E.request_bytes("m", 1, d, key=target)
    carries = {S.example_rounds(w)[1] for w in ROUNDS}
    assert carries == {0, 1, 2}


def emit_outcome(d):
    """what ex_emit does with a Classify request of input dict d, from the host plan of its columns and its real example sizes"""
    q = E.ReqPlan("m", 1, d)
    E.plan([q])
    sizes, _ = E.example_bytes(d)
    out = E.emit(q, sizes)
    assert E.covers_once(q, sizes, out["stores"])
    return out


def one_string_examples(lens, start, seed):
    rng = np.random.default_rng(seed)
    strs = [rng.integers(0, 256, L, dtype=np.uint8).tobytes() for L in lens]
    return {"s": bytes_column(strs, (len(strs),), start=start), "i": np.arange(len(strs), dtype=np.int64)}


def test_example_strings_around_the_emit_image(codec):
    """string bytes ending exactly at a kExStage image edge, straddling one at several phases (a partial vector carried to the
    next batch), and examples larger than the image (written in place)"""
    cases = {}
    for start in (0, 1, 15):
        cases["straddle%d" % start] = one_string_examples([S.K_STAGE // 5 + 37 * k for k in range(12)], start, start)
    cases["big"] = one_string_examples([3 * S.K_STAGE + 5, 40, S.K_STAGE + 1], 3, 4)
    # exact: the string length whose example ends on the image's last byte
    exact = next(d for L in range(S.K_STAGE - 64, S.K_STAGE) for d in [one_string_examples([L], 0, 5)] if emit_outcome(d)["full"])
    cases["exact"] = exact
    seen = {}
    for name, d in cases.items():
        got = codec.encode_example_requests([("m", 1, d)])[0]
        same(got, E.request_bytes("m", 1, d), name)
        seen[name] = emit_outcome(d)
    assert seen["exact"]["full"] >= 1
    assert all(seen["straddle%d" % st]["carried"] for st in (0, 1, 15))
    assert seen["big"]["in_place"] and any(b - a > S.K_STAGE for a, b in seen["big"]["stores"])


def test_example_context_of_more_than_32_strings(codec):
    """an ExampleListWithContext whose bytes context takes two and three 32-string rounds, beside bytes examples"""
    dist = distinct(SHORT_LENS + [300], 26)
    rng = np.random.default_rng(27)
    d = {"s": bytes_column([dist[i] for i in rng.integers(0, len(dist), 4 * 33)], (4, 33), start=5),
         "x": np.ones((4, 2), np.float32)}
    for m in (33, 65, 96):
        ctx = {"c": bytes_column([dist[i] for i in rng.integers(0, len(dist), m)], None, start=m % 16),
               "one": bytes_column([b"\x00q"], ()), "i": np.arange(3)}
        assert S.example_rounds(m)[1] >= 1
        for key in (None, "elwc"):
            kw = {} if key is None else {"predict_input": key}
            got = codec.encode_example_requests([("m", 1, d, ctx)], **kw)[0]
            same(got, E.request_bytes("m", 1, d, key=key, context=ctx), (m, key))
