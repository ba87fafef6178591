"""The mutant corpus (tests/decode_mutants.py) through every device decode route, against the host build of the tag walker
and the reference.

Records lie back to back in one arena at offsets that take every residue mod 128 (the device walk reads through a two-line,
128-byte cache), with 256 bytes of headroom on both sides; a truncated record keeps its real continuation bytes behind it.
The single-launch decode runs every batch twice on a fresh context: the first launch walks every record and learns the
template of record 0 (the clean seed), the second serves the records that carry the seed's framing from that template.
Which records those are is predicted by a restatement of the verdict (decode_mutants.verdict), and the context's path
counters must show exactly that split.  Every destination slot is filled with 0xEE first, and every byte outside the
ranges of the outputs a record decoded must still hold it afterwards.
"""
import ctypes as C
import os
from collections import Counter

import ml_dtypes
import numpy as np
import pytest
from google.protobuf.message import DecodeError

import decode_mutants as D
from devutil import Dev
from min_tfs_client import _native as N
from oracle import ref_port, wire_oracle

pytestmark = pytest.mark.gpu

CORPUS = D.corpus()
RESP = [(s, ms) for s, ms in CORPUS if not s.tensor]
TENS = [(s, ms) for s, ms in CORPUS if s.tensor]
NP16 = {19: np.float16, 14: ml_dtypes.bfloat16}
COUNTS = Counter()      # what the corpus exercised, reported at the end of the module


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\ncoverage:", dict(sorted(COUNTS.items())))


_walks = {}


def walk(m, **kw):
    k = (m.buf, m.rec_len, m.tensor, tuple(sorted(kw.items())))
    if k not in _walks:
        _walks[k] = D.walk(m.buf, m.rec_len, tensor=m.tensor, **kw)
    return _walks[k]


def seed_mutant(s):
    return D.Mutant(s.name, "seed", s.wire, len(s.wire), s.tensor)


def place(recs):
    """One arena holding every record's buffer back to back, record i at an offset == i (mod 128), 256 B of headroom."""
    offs, cur = [], 256
    for i, m in enumerate(recs):
        cur += (i - cur) % 128
        offs.append(cur)
        cur += len(m.buf)
    arena = np.zeros(cur + 256, dtype=np.uint8)
    for o, m in zip(offs, recs):
        arena[o: o + len(m.buf)] = np.frombuffer(m.buf, dtype=np.uint8)
    n = len(recs)
    COUNTS["line phases"] = max(COUNTS["line phases"], len({o % 128 for o in offs}))
    return arena, (C.c_uint64 * n)(*offs), (C.c_uint64 * n)(*[m.rec_len for m in recs])


def fields(o):
    """The fields of a table entry that carry meaning (the inline arrays only up to rank / n_inline)."""
    return (int(o.key_off), int(o.key_len), int(o.dtype), int(o.rank), int(o.flags), int(o.value_field), int(o.n_runs),
            tuple(int(o.dims[k]) for k in range(min(o.rank, N.MAX_RANK))),
            tuple((int(r.off), int(r.len), int(r.count), int(r.stride), int(r.field)) for r in (o.runs[k] for k in range(o.n_inline))),
            int(o.content_off), int(o.content_len), int(o.msg_off), int(o.msg_len), int(o.n_elems), int(o.dst_bytes), int(o.n_strings),
            int(o.dst_off), int(o.status), int(o.n_inline), int(o.spill_seq))


def _chunks(lst, k):
    return [lst[i: i + k] for i in range(0, len(lst), k)]


# ---- two-phase parse + unpack ---------------------------------------------------------------------------------------------
def _check_parse(dev, m, i, status, n_outs, outs, spec, max_outputs=16):
    w = walk(m)
    what = (m.seed, m.kind, m.rec_len)
    assert status == w.status, (what, status, w.status)
    if w.status != N.OK:
        return
    got = [outs[i * max_outputs + k] for k in range(n_outs)] if not m.tensor else [outs[i]]
    assert len(got) == len(w.outs), what
    for k, (g, e) in enumerate(zip(got, w.outs)):
        assert g.spill_rec == i, what
        assert fields(g) == fields(e), (what, k)
        if g.flags & N.OF_SPILLED:
            dims, runs = (C.c_int64 * g.rank)(), (N.Run * g.n_runs)()
            N.check(dev.lib.b200tfs_output_dims(dev.ctx, C.byref(g), dims, g.rank))
            N.check(dev.lib.b200tfs_output_runs(dev.ctx, C.byref(g), runs, g.n_runs))
            assert list(dims) == w.dims[k] and [(r.off, r.len, r.count, r.stride, r.field) for r in runs] == w.runs[k], what
            COUNTS["spilled outputs read back"] += 1
    if not m.tensor:
        assert D.spec_text(m.record, spec) == D.spec_text(m.record, w.spec), what


def _free(dev, p):
    dev.lib.b200tfs_free(dev.ctx, p)
    dev.allocs.remove(p)


def _parse(dev, recs, host, tensor):
    arena, off, ln = place(recs)
    n = len(recs)
    status = (C.c_int32 * n)()
    if tensor:
        outs = (N.Output * n)()
        n_outs, specs = None, None
        if host:
            N.check(dev.lib.b200tfs_parse_tensor_protos_host(dev.ctx, arena.ctypes.data, n, off, ln, outs, status))
        else:
            arena_dev = dev.upload(arena)
            N.check(dev.lib.b200tfs_parse_tensor_protos(dev.ctx, arena_dev, n, off, ln, outs, status))
            _free(dev, arena_dev)
        return arena, off, outs, [1] * n, [None] * n, status, None
    outs, n_outs, specs = (N.Output * (n * 16))(), (C.c_int32 * n)(), (N.ModelSpec * n)()
    arena_dev = None
    if host:
        N.check(dev.lib.b200tfs_parse_responses_host(dev.ctx, arena.ctypes.data, n, off, ln, 16, outs, n_outs, specs, status))
    else:
        arena_dev = dev.upload(arena)
        N.check(dev.lib.b200tfs_parse_responses(dev.ctx, arena_dev, n, off, ln, 16, outs, n_outs, specs, status))
    return arena, off, outs, n_outs, specs, status, arena_dev


def _reference_outputs(m):
    """tensor_proto_to_ndarray per output over the protobuf runtime: key -> array or exception class; None: the runtime
    refuses the record."""
    from tensorflow.core.framework import tensor_pb2
    from tensorflow_serving.apis import predict_pb2

    try:
        msg = (tensor_pb2.TensorProto if m.tensor else predict_pb2.PredictResponse).FromString(m.record)
    except DecodeError:
        return None
    got = {}
    for key, tp in ([("", msg)] if m.tensor else msg.outputs.items()):
        try:
            got[key] = ref_port.from_tensor_proto(tp)
        except Exception as e:     # noqa: BLE001 - the class is what is compared
            got[key] = type(e)
    return got


def _unpack_and_check(dev, recs, arena_dev, off, outs, n_outs, status, per):
    """b200tfs_unpack_outputs for every OK output of every OK record (fixed-width and varint), into one canary-filled buffer."""
    jobs = []
    for i, m in enumerate(recs):
        if status[i] != N.OK:
            continue
        for k in range(n_outs[i]):
            o = outs[i * per + k]
            if o.status == N.OK and o.n_elems and o.dtype != 7:
                jobs.append((i, k, o))
    if not jobs:
        return
    at, total = [], 0
    for _, _, o in jobs:
        at.append(total + 64)
        total = (total + 64 + int(o.dst_bytes) + 255) & ~255
    total += 256
    base = dev.malloc(total)
    N.check(dev.lib.b200tfs_memset(dev.ctx, base, 0xEE, total))
    mm = len(jobs)
    t = (N.Output * mm)(*[o for _, _, o in jobs])
    dst = (C.c_void_p * mm)(*[base + a for a in at])
    codes = (C.c_int32 * mm)(*[o.dtype for _, _, o in jobs])
    st = (C.c_int32 * mm)()
    N.check(dev.lib.b200tfs_unpack_outputs(dev.ctx, arena_dev, mm, t, (C.c_uint64 * mm)(*[off[i] for i, _, _ in jobs]), dst, codes, st))
    got = dev.download(base, total)
    mask = np.zeros(total, dtype=bool)
    refs = {}
    for j, (i, k, o) in enumerate(jobs):
        m = recs[i]
        what = (m.seed, m.kind, m.rec_len, k)
        if i not in refs:
            refs[i] = _reference_outputs(m)
        ref = refs[i]
        raw = got[at[j]: at[j] + o.dst_bytes].tobytes()
        if st[j] == N.OK:
            mask[at[j]: at[j] + o.dst_bytes] = True
            COUNTS["unpacked outputs"] += 1
        else:
            COUNTS["unpack errors"] += 1
        if ref is None:
            # the runtime refuses the record although the walk accepted it: only a malformed packed varint gets here
            # (test_decode_mutants_cpu.py), and unpacking that output must report it
            assert st[j] != N.OK or not D.malformed_varints(m.buf, walk(m), k), what
            if st[j] == N.OK and o.dtype in D.FIXED:
                assert raw == D.fixed_values(m.buf, walk(m), k), what
            continue
        want = ref["" if m.tensor else m.record[o.key_off: o.key_off + o.key_len].decode()]
        if st[j] == N.OK:
            assert isinstance(want, np.ndarray), (what, want)     # never OK with values where the reference raises
            if o.dtype in D.FIXED:
                assert raw == D.fixed_values(m.buf, walk(m), k) == want.tobytes(), what
            else:
                assert raw == want.tobytes(), what
        else:
            assert isinstance(want, type), (what, st[j])
    assert (got[~mask] == 0xEE).all(), "unpack stored outside its outputs"
    _free(dev, base)


@pytest.mark.parametrize("host", [False, True], ids=["device", "host"])
def test_parse_and_unpack_every_mutant(host):
    """b200tfs_parse_responses[_host] (max_outputs 16, spill re-run) equals the host walker field for field; every OK output
    unpacks to the reference's values, and an output the reference refuses never unpacks OK."""
    dev = Dev(0)
    try:
        for s, ms in RESP + TENS:
            recs = [seed_mutant(s)] + ms
            for batch in _chunks(recs, 4096):
                arena, off, outs, n_outs, specs, status, arena_dev = _parse(dev, batch, host, s.tensor)
                for i, m in enumerate(batch):
                    _check_parse(dev, m, i, status[i], n_outs[i], outs, specs[i] if specs is not None else None)
                if not host and not s.tensor:
                    _unpack_and_check(dev, batch, arena_dev, off, outs, n_outs, status, 16)
                if arena_dev is not None:      # one batch's arena on the device at a time
                    _free(dev, arena_dev)
                COUNTS["parsed records"] += len(batch)
    finally:
        dev.close()


# ---- the single-launch decode ---------------------------------------------------------------------------------------------
def _stats(dev):
    a, b, c = C.c_uint64(), C.c_uint64(), C.c_uint64()
    N.check(dev.lib.b200tfs_decode_stats(dev.ctx, C.byref(a), C.byref(b), C.byref(c)))
    return a.value + b.value, c.value


def _launches(dev):
    v = C.c_uint64()
    N.check(dev.lib.b200tfs_kernel_launches(dev.ctx, C.byref(v)))
    return v.value


def _stride(recs):
    return (max(m.rec_len for m in recs) + 256 * (N.FUSED_MAX_OUTPUTS + 1) + 255) & ~255


def _fused(dev, recs, stride, host=False):
    """One b200tfs_decode_responses (device wire) or b200tfs_decode_responses_host_async (pinned host wire) over recs."""
    arena, off, ln = place(recs)
    n = len(recs)
    keep = []
    if host:
        wire = N.PinnedBuffer(arena.size)
        wire.array[:] = arena
        out = N.PinnedBuffer(stride * n)
        out.array[:] = 0xEE
        keep += [wire, out]
        N.check(dev.lib.b200tfs_decode_responses_host_async(dev.ctx, wire.ptr, n, off, ln, out.ptr, stride))
    else:
        dst = dev.malloc(stride * n)
        N.check(dev.lib.b200tfs_memset(dev.ctx, dst, 0xEE, stride * n))
        N.check(dev.lib.b200tfs_decode_responses(dev.ctx, dev.upload(arena), n, off, ln, dst, stride))
    outs = (N.Output * (n * N.FUSED_MAX_OUTPUTS))()
    n_outs, specs, status = (C.c_int32 * n)(), (N.ModelSpec * n)(), (C.c_int32 * n)()
    N.check(dev.lib.b200tfs_decode_results(dev.ctx, n, outs, n_outs, specs, status))
    slots = (out.array.copy() if host else dev.download(dst, stride * n)).reshape(n, stride)
    for p in keep:
        p.free()
    if not host:
        dev.lib.b200tfs_free(dev.ctx, dst)
        dev.allocs.remove(dst)
        dev.lib.b200tfs_free(dev.ctx, dev.allocs.pop())
    return slots, outs, n_outs, specs, status


def _check_fused(recs, stride, result, cast=0, tpl=None):
    """Status, table, values and destination canary of every record of one single-launch decode."""
    slots, outs, n_outs, specs, status = result
    K = N.FUSED_MAX_OUTPUTS
    for i, m in enumerate(recs):
        what = (m.seed, m.kind, m.rec_len, i)
        w = walk(m, max_outputs=K, spill=False)
        want = N.E_NONCANONICAL if w.status == N.E_SPILL else w.status
        slot = slots[i]
        if status[i] == N.E_NONCANONICAL and want == N.OK:
            # a record of the template's length but other framing whose values need more tiles than the template's:
            # reported, not decoded (the two-phase route decodes it: test_parse_and_unpack_every_mutant)
            assert tpl is not None and m.rec_len == tpl.rec_len, what
            assert (slot == 0xEE).all(), what
            COUNTS["noncanonical same-length records"] += 1
            continue
        assert status[i] == want, (what, status[i], want)
        if want != N.OK:
            assert (slot == 0xEE).all(), ("a record that did not decode wrote into its slot", what)
            continue
        exp = D.layout(w.outs, stride, cast)
        assert n_outs[i] == len(exp), what
        mask = np.zeros(stride, dtype=bool)
        for k, e in enumerate(exp):
            g = outs[i * K + k]
            assert fields(g) == fields(e), (what, k)
            if e.status == N.OK and e.n_elems and e.dtype in D.FIXED:
                got = slot[e.dst_off: e.dst_off + e.dst_bytes].tobytes()
                vals = D.fixed_values(m.buf, w, k)
                if cast and e.dtype == 1:
                    vals = wire_oracle.narrow_f32(np.frombuffer(vals, np.float32), NP16[cast]).tobytes()
                assert got == vals, (what, k)
                mask[e.dst_off: e.dst_off + e.dst_bytes] = True
        assert D.spec_text(m.record, specs[i]) == D.spec_text(m.record, w.spec), what
        assert (slot[~mask] == 0xEE).all(), ("a store outside the outputs' ranges", what)


def _predicted(tpl, recs):
    return sum(1 for m in recs if tpl is not None and D.verdict(tpl, m.buf, m.rec_len))


def _same_length(s, ms):
    return [m for m in ms if m.rec_len == len(s.wire)]


def _spread(s, ms, n):
    """About n same-length mutants for the small batches: every same-length framing edit, then framing-bit flips spread
    over the whole record and a few value flips."""
    same = _same_length(s, ms)
    edits = [m for m in same if m.kind.startswith("same_len")]
    flips = [m for m in same if m.kind == "framing_flip"]
    values = [m for m in same if m.kind == "value_flip"]
    rest = flips[:: max(len(flips) // max(n - len(edits) - 4, 1), 1)] + values[:: max(len(values) // 4, 1)][:4]
    return edits + rest[: max(n - len(edits), 0)]


def _twice(dev, recs, label, host=False, cast=0, fresh=False):
    """The same batch (record 0: the clean seed) twice.  The second launch is served by the template the first one left of
    record 0: its split between template and walk must be the predicted one.  On a fresh context the first launch walks
    every record - unless the host walked record 0 itself (host-resident wire), which makes it the predicted split too.
    Returns how many same-length records with other framing the second launch's verdict refused."""
    s_len = recs[0].rec_len
    tpl = D.template_of(recs[0].record)
    stride = _stride(recs)
    hits = _predicted(tpl, recs)
    for rep in range(2):
        t0, w0 = _stats(dev)
        res = _fused(dev, recs, stride, host)
        t1, w1 = _stats(dev)
        _check_fused(recs, stride, res, cast, tpl)
        split = (t1 - t0, w1 - w0)
        if rep == 1:
            assert split == (hits, len(recs) - hits), (label, recs[0].seed, rep, split, hits)
            refused = sum(1 for m in recs if m.rec_len == s_len and m.kind != "value_flip" and not D.verdict(tpl, m.buf, m.rec_len)) if tpl else 0
            COUNTS[f"same-length framing mutants refused by the verdict ({label})"] += refused
            COUNTS[f"records served by the template ({label})"] += hits
        elif fresh:
            assert split == (0, len(recs)) or (host and split == (hits, len(recs) - hits)), (label, recs[0].seed, rep, split)
        if len(recs) > 16:
            COUNTS[f"batches on the cta_rec path ({label})"] += 1
    return refused


def _fresh(env=None):
    old = {k: os.environ.get(k) for k in (env or {})}
    os.environ.update(env or {})
    try:
        return Dev(0)
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v


ROUTES = {
    "device": None,                                         # template in the parameters once the host adopted it
    "device_template": {"B200TFS_NO_INLINE_TEMPLATE": "1"},  # the per-warp verdict reads the template from device memory
    "staged": {"B200TFS_TILE_BYTES": "65536"},               # fat tiles select the staged kernel: per-CTA verdict
    "host": None,                                           # host-resident wire: the host walks record 0 itself
}


@pytest.mark.parametrize("route", list(ROUTES))
def test_single_launch_decode_of_every_mutant(route):
    """device / device_template: decode_fused_kernel, whose per-warp verdict reads the template from the kernel parameters /
    from device memory; staged: 64 KB tiles select decode_fused_staged_kernel (per-CTA verdict); host:
    b200tfs_decode_responses_host_async (the host walks record 0 and hands the template over in the parameters).  Each over
    the whole corpus of each seed (a batch on the cta_rec table path) and over small batches of same-length mutants (records
    in the parameters, one 32 KB tile per CTA: on every route but `staged`, the per-warp verdict)."""
    host = route == "host"
    refused = evicting = 0
    phases = set()
    for s, ms in RESP:
        seed = seed_mutant(s)
        dev = _fresh(ROUTES[route])
        try:
            _twice(dev, [seed] + ms, route, host=host, fresh=True)
            phases.update(range(min(len(ms) + 1, 128)))
            for batch in _chunks(_spread(s, ms, 60), 15):
                refused += _twice(dev, [seed] + batch, route, host=host)
            value = np.zeros(len(s.wire), dtype=bool)
            for a, b in D.value_ranges(walk(seed)):
                value[a:b] = True
            if len({int(q) >> 7 for q in np.flatnonzero(~value)}) >= 3:     # at any phase, three lines: one eviction at least
                evicting += 1
        finally:
            dev.close()
    verdict = "per-CTA" if route == "staged" else "per-warp"
    COUNTS[f"same-length framing mutants refused by the {verdict} verdict in small batches ({route})"] += refused
    COUNTS[f"seeds whose device walk evicts cache lines ({route})"] += evicting
    # what this route is there to exercise must stay in the corpus
    assert refused >= 100 and evicting >= 2 and len(phases) == 128, (refused, evicting, len(phases))
    assert COUNTS[f"batches on the cta_rec path ({route})"] >= len(RESP)


def test_sliced_host_decode_of_single_large_mutants():
    """b200tfs_set_pipeline(ctx, 4096, 4): one large response per call takes the sliced, trusted path (the host built the
    template from the record's own bytes); records that do not qualify take the plain call."""
    dev = Dev(0)
    try:
        N.check(dev.lib.b200tfs_set_pipeline(dev.ctx, 4096, 4))
        p0 = C.c_uint64()
        N.check(dev.lib.b200tfs_pipelined_calls(dev.ctx, C.byref(p0)))
        n = 0
        for s, ms in RESP:
            if len(s.wire) < 65536:
                continue
            pick = [seed_mutant(s)] + [m for m in ms if m.kind.startswith("same_len")] + [m for m in ms if m.kind == "value_flip"][:24] \
                + [m for m in ms if m.kind in ("truncate", "framing_flip")][::40]
            for m in pick:
                stride = _stride([m])
                _check_fused([m], stride, _fused(dev, [m], stride, host=True))
                n += 1
        p1 = C.c_uint64()
        N.check(dev.lib.b200tfs_pipelined_calls(dev.ctx, C.byref(p1)))
        assert p1.value - p0.value >= 20, (p0.value, p1.value, n)
        COUNTS["sliced single-record decodes"] += p1.value - p0.value
    finally:
        dev.close()


@pytest.mark.parametrize("cast", [19, 14])
def test_narrowing_decode_of_same_length_mutants(cast):
    """b200tfs_set_decode_cast: one response per launch, small batches, and a >= 4 MiB batch of records of one length, which
    runs as three launches (mode-1 verify -> guard[r] -> move_guarded_kernel -> mode 2)."""
    mode1 = 0
    for s, ms in RESP:
        seed = seed_mutant(s)
        same = _same_length(s, ms)
        dev = Dev(0)
        try:
            N.check(dev.lib.b200tfs_set_decode_cast(dev.ctx, cast))
            tpl = D.template_of(s.wire)
            stride = _stride([seed] + same)
            _check_fused([seed], stride, _fused(dev, [seed], stride), cast, tpl)
            cur = tpl            # the template of the previous launch's record 0 (a walked record 0 replaces it)
            for m in [x for x in same if x.kind.startswith("same_len")] + same[:: max(len(same) // 12, 1)]:
                t0, w0 = _stats(dev)
                _check_fused([m], stride, _fused(dev, [m], stride), cast, cur)
                t1, _ = _stats(dev)
                hit = _predicted(cur, [m])
                assert t1 - t0 == hit, (s.name, m.kind)
                COUNTS[f"single responses served by the template (cast {cast})"] += hit
                if not hit:
                    cur = D.template_of(m.record)
            for batch in _chunks(_spread(s, ms, 45), 15):
                _twice(dev, [seed] + batch, f"cast {cast}", cast=cast)
            if tpl is not None and len(s.wire) * 60 >= 4 << 20 and any(not v for _, _, v in tpl.chunks):
                batch = [seed] + [x for x in same if x.kind.startswith("same_len")] + [x for x in same if x.kind == "value_flip"]
                batch += [x for x in same if x.kind not in ("value_flip",) and not x.kind.startswith("same_len")]
                batch = batch[:64]
                assert len(batch) * len(s.wire) >= 4 << 20
                stride = _stride(batch)
                _fused(dev, [seed] * len(batch), stride)            # the context learns the record length
                l0, (t0, w0) = _launches(dev), _stats(dev)
                _check_fused(batch, stride, _fused(dev, batch, stride), cast, tpl)
                t1, w1 = _stats(dev)
                hits = _predicted(tpl, batch)
                assert _launches(dev) - l0 == 3, "verify, guarded move, fallback"
                assert (t1 - t0, w1 - w0) == (hits, len(batch) - hits), s.name
                COUNTS[f"records judged by the mode-1 verify launch (cast {cast})"] += len(batch)
                COUNTS[f"same-length mutants refused by the mode-1 verify launch (cast {cast})"] += len(batch) - hits
                mode1 += len(batch) - hits
        finally:
            dev.close()
    assert mode1 >= 4, mode1


@D.EXHAUSTIVE
def test_every_value_flip_of_the_large_seeds(request):
    """Every single-bit flip of every value byte of the large seeds (some 640 000 records per seed), in batches of 512:
    the two-phase parse + unpack and the single-launch decode (walk, then template) as above."""
    D.require_exhaustive(request.config)
    dev = Dev(0)
    try:
        for s, _ in RESP + TENS:
            if len(s.wire) <= D.SMALL:
                continue
            flips = D.value_flips(s)
            while True:
                batch = [seed_mutant(s)] + [m for _, m in zip(range(511), flips)]
                if len(batch) == 1:
                    break
                arena, off, outs, n_outs, specs, status, arena_dev = _parse(dev, batch, False, s.tensor)
                for i, m in enumerate(batch):
                    _check_parse(dev, m, i, status[i], n_outs[i], outs, specs[i] if specs is not None else None)
                if not s.tensor:
                    _unpack_and_check(dev, batch, arena_dev, off, outs, n_outs, status, 16)
                    _twice(dev, batch, "exhaustive")
                if arena_dev is not None:
                    _free(dev, arena_dev)
                _walks.clear()
    finally:
        dev.close()


# ---- the Python codec on top ----------------------------------------------------------------------------------------------
def _codec_reference(rec, strict):
    """What the reference gives for one response: ref_port (strict) or the oracle's tolerant decode - a dict of arrays, or
    the classes of the exceptions it may raise (a malformed message: DecodeError).  When several outputs fail, which one
    the reference reports first follows the runtime's map iteration order, which nothing specifies: any of them is right."""
    try:
        return ref_port.decode_predict_response(rec) if strict else wire_oracle.decode_predict_response(rec, strict=False)
    except (DecodeError, wire_oracle.ParseError):
        return (DecodeError,)
    except Exception as e:      # noqa: BLE001 - the class is what is compared
        if not strict:
            return (type(e),)
    from tensorflow_serving.apis import predict_pb2

    raised = set()
    for tp in predict_pb2.PredictResponse.FromString(rec).outputs.values():
        try:
            ref_port.from_tensor_proto(tp)
        except Exception as e:  # noqa: BLE001
            raised.add(type(e))
    return tuple(raised)


def _codec_mismatch(got, want):
    """None when the codec's answer equals the reference's, else a short description."""
    if isinstance(want, tuple):
        return None if isinstance(got, type) and issubclass(got, want) else \
            f"want {[w.__name__ for w in want]}, got {got if isinstance(got, type) else 'arrays'}"
    if isinstance(got, type):
        return f"want arrays, got {got.__name__}"
    if sorted(got) != sorted(want):
        return f"keys {sorted(got)} != {sorted(want)}"
    for k, b in want.items():
        a = got[k]
        if a.dtype != b.dtype or a.shape != b.shape:
            return f"{k}: {a.dtype}{a.shape} != {b.dtype}{b.shape}"
        if (D.quiet_f32(a.tobytes()) if a.dtype == np.float32 else a.tobytes()) != (D.quiet_f32(b.tobytes()) if b.dtype == np.float32 else b.tobytes()):
            return f"{k}: values differ"
    return None


def _codec_call(codec, recs, strict):
    try:
        return [r[0] for r in codec.decode_predict_responses(recs, strict=strict)], None
    except Exception as e:      # noqa: BLE001
        return None, e


@pytest.mark.parametrize("strict", [True, False], ids=["strict", "tolerant"])
def test_codec_decode_of_every_mutant(codec, strict):
    """Codec.decode_predict_responses over the whole corpus: the arrays ref_port (strict=True) / the oracle's tolerant decode
    (strict=False) give, or the same exception class.  Records the reference accepts go in batches of up to 64 (a batch
    whose records all decode takes the single launch, else the two-phase path); a record the reference refuses goes alone,
    since one refused record fails its whole batch.  The oracle does not decode string outputs, so the tolerant pass skips
    the seed that has one."""
    bad, n = [], 0
    for s, ms in RESP:
        if not strict and s.name == "multi":
            continue
        recs = [seed_mutant(s)] + ms
        want = [_codec_reference(m.record, strict) for m in recs]
        ok = [i for i, w in enumerate(want) if not isinstance(w, tuple)]
        singles = [i for i, w in enumerate(want) if isinstance(w, tuple)]
        for batch in _chunks(ok, 64):
            got, err = _codec_call(codec, [recs[i].record for i in batch], strict)
            if got is None:
                singles += batch            # find which record it was
                continue
            for i, g in zip(batch, got):
                why = _codec_mismatch(g, want[i])
                if why:
                    bad.append((recs[i].seed, recs[i].kind, recs[i].rec_len, why))
        for i in singles:
            got, err = _codec_call(codec, [recs[i].record], strict)
            why = _codec_mismatch(got[0] if got else type(err), want[i])
            if why:
                bad.append((recs[i].seed, recs[i].kind, recs[i].rec_len, why, f"{type(err).__name__}: {err}" if err else ""))
        n += len(recs)
    COUNTS[f"codec decodes ({'strict' if strict else 'tolerant'})"] += n
    assert not bad, (len(bad), bad[:40])


def test_codec_strict_rank0_raises_type_error_whatever_the_values(codec):
    """A rank-0 output (its shape field lost, as a framing-bit flip of the f32 seed does): tensor_proto_to_ndarray calls
    reshape() with no dims, a TypeError whatever the element count.  The codec used to raise the element count's ValueError
    first whenever there was not exactly one value."""
    x = D.f32(7, 1)
    for n in (0, 1, 7):
        rec = D.out("scores", 1, [], D.ld(0x2A, x[:n].tobytes())) + D.mspec()
        with pytest.raises(TypeError):
            ref_port.decode_predict_response(rec)
        with pytest.raises(TypeError):
            codec.decode_predict_responses([rec], strict=True)
