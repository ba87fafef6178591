"""The Classify / Regress / MultiInference decode on the GPU at every window, stage and chain edge of the warp entry finder
(tests/xr_edges.py builds the cases; tests/test_example_response_edges_cpu.py shows that they reach those edges).  The records lie
in a device arena at chosen residues of their address (mod 16: staging; mod 128: the cursors' lines), through the device-arena
entry points, the _host_async forms and the Python route.  Every case against the definition (FromString): per-record status,
rows and first row, the batch words, values / scores bit for bit, labels as bytes, model_spec; and every destination byte past
the used rows still holds its canary."""
import ctypes as C

import numpy as np
import pytest
from google.protobuf.message import DecodeError

import example_response_corpus as X
import multi_inference_corpus as M
import xr_edges as E
from devutil import Dev
from min_tfs_client import _native as N

pytestmark = pytest.mark.gpu
CANARY = 0xA5A5A5A5
RESIDUES = list(range(16)) + [17, 50, 63, 64, 100, 127]


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _place(wires, residues):
    """(image, offsets): every record at an offset with the given residue mod 128"""
    offs, cur = [], 0
    for w, r in zip(wires, residues):
        at = ((cur + 127) & ~127) + r
        offs.append(at)
        cur = at + len(w)
    img = np.zeros(cur + 256, np.uint8)
    for w, at in zip(wires, offs):
        img[at: at + len(w)] = np.frombuffer(w, np.uint8)
    return img, offs


def _spec_ok(wire, s, ms):
    text = lambda off, n: wire[off: off + n].decode("utf-8")   # noqa: E731
    return (text(s.name_off, s.name_len) == ms.name and text(s.signature_off, s.signature_len) == ms.signature_name
            and bool(s.has_version) == ms.HasField("version") and (not s.has_version or s.version == ms.version.value)
            and text(s.label_off, s.label_len) == ms.version_label)


def _definition(kind, wire):
    """('ok', values [rows(, C)], labels, model_spec) or ('parse',)"""
    from tensorflow_serving.apis.classification_pb2 import ClassificationResponse
    from tensorflow_serving.apis.regression_pb2 import RegressionResponse

    try:
        vals, labels, _ = X.expected(kind, [wire])
    except DecodeError:
        return ("parse",)
    ms = (RegressionResponse if kind == X.REGRESS else ClassificationResponse).FromString(wire).model_spec
    return ("ok", vals, labels, ms)


def decode_batch(dev, kind, wires, residues, host_async=False, values_cap=None, labels_cap=None):
    """Run one batch; returns (per [n, 3], specs, batch, values (all of the buffer), label refs (all of it), image, offsets, caps)"""
    lib = dev.lib
    n = len(wires)
    img, offs = _place(wires, residues)
    off = (C.c_uint64 * n)(*offs)
    ln = (C.c_uint64 * n)(*[len(w) for w in wires])
    mr, mv = C.c_uint64(), C.c_uint64()
    N.check(lib.b200tfs_example_response_bound(kind, n, ln, C.byref(mr), C.byref(mv)))
    bound = int(mv.value)
    vcap = bound if values_cap is None else values_cap
    lcap = (bound if labels_cap is None else labels_cap) if kind == X.CLASSIFY else 0
    room = bound + 64
    v = dev.upload(np.full(room, CANARY, np.uint32))
    lab = dev.upload(np.full(2 * room, CANARY, np.uint32))
    per, specs, batch = (C.c_int64 * (3 * n))(), (N.ModelSpec * n)(), (C.c_int64 * 5)()
    if host_async:
        N.check(lib.b200tfs_decode_example_responses_host_async(dev.ctx, kind, img.ctypes.data, n, off, ln, v, vcap,
                                                                lab if kind == X.CLASSIFY else None, lcap))
    else:
        arena = dev.upload(img)
        N.check(lib.b200tfs_decode_example_responses(dev.ctx, kind, arena, n, off, ln, v, vcap, lab if kind == X.CLASSIFY else None, lcap))
    N.check(lib.b200tfs_example_response_results(dev.ctx, n, per, specs, batch))
    got_v = dev.download(v, 4 * room, np.uint32)
    got_l = dev.download(lab, 8 * room, np.uint32).reshape(-1, 2)
    return np.array(per, np.int64).reshape(n, 3), specs, list(batch), got_v, got_l, img, offs, (vcap, lcap)


def check_batch(dev, kind, wires, residues, index_errors=(), host_async=False):
    """Decode the batch and hold every record against the definition; returns the per-record outcomes"""
    per, specs, batch, vals, refs, img, offs, _ = decode_batch(dev, kind, wires, residues, host_async)
    defs = [_definition(kind, w) for w in wires]
    C_ = 0
    if kind == X.CLASSIFY:   # C: the batch's first response with rows sets it, a malformed one included
        i0 = next((i for i, d in enumerate(defs) if d[0] == "ok" and len(d[1])), None)
        C_ = defs[i0][1].shape[1] if i0 is not None else int(batch[1])
        if i0 is not None and any(int(per[i, 1]) for i in range(i0)):
            C_ = int(batch[1])
    row = 0
    bad = None
    for i, (w, d) in enumerate(zip(wires, defs)):
        st, r0, rows = int(per[i, 2]), int(per[i, 0]), int(per[i, 1])
        assert r0 == row, (i, r0, row)
        row += rows
        if d[0] == "parse":
            assert st == N.E_PARSE, (i, st, w[:64].hex())
            if i in index_errors:
                assert rows == 0, i
        else:
            assert st == N.OK, (i, st)
            assert rows == len(d[1]), (i, rows, len(d[1]))
            if kind == X.REGRESS:
                assert np.array_equal(vals[r0: r0 + rows], _bits(d[1])), i
            else:
                assert not rows or d[1].shape[1] == C_, i
                assert np.array_equal(vals[r0 * C_: (r0 + rows) * C_], _bits(d[1]).ravel()), i
                got = [[img[offs[i] + int(refs[(r0 + j) * C_ + k, 0]): offs[i] + int(refs[(r0 + j) * C_ + k, 0]) + int(refs[(r0 + j) * C_ + k, 1])]
                        .tobytes() for k in range(C_)] for j in range(rows)]
                assert got == [[lab.encode() for lab in r] for r in d[2]], i
            assert _spec_ok(w, specs[i], d[3]), i
        if st != N.OK and bad is None:
            bad = (st, i)
    per_row = C_ if kind == X.CLASSIFY else 1
    assert batch[0] == row and batch[1] == C_
    assert batch[3] == (bad[0] if bad else N.OK) and batch[4] == (bad[1] if bad else -1)
    if kind == X.CLASSIFY and not bad:
        labels = [r for d in defs for r in d[2]]
        assert batch[2] == int(all(r == labels[0] for r in labels))
    assert (vals[row * per_row:] == CANARY).all(), "a value store past the used rows"
    assert (refs[row * per_row:] == CANARY).all(), "a label store past the used rows"
    return defs


@pytest.fixture(scope="module")
def dev():
    d = Dev()
    yield d
    d.close()


def test_regress_grid_at_every_residue(dev):
    """Window, chain, stage and error cases, the whole grid in one batch per residue of the record address."""
    for k, rec in enumerate(RESIDUES):
        cases = E.regress_grid(rec)
        errs = {i for i, c in enumerate(cases) if c.name.startswith("err_")}
        check_batch(dev, X.REGRESS, [c.wire for c in cases], [rec] * len(cases), errs, host_async=k % 2 == 1)


def test_regress_grid_at_mixed_residues(dev):
    cases = E.regress_grid()
    wires = [c.wire for c in cases] + [w for _, w in E.emit_cases()]
    res = [RESIDUES[i % len(RESIDUES)] for i in range(len(wires))]
    check_batch(dev, X.REGRESS, wires, res, {i for i, c in enumerate(cases) if c.name.startswith("err_")})


def test_long_tags_through_the_kernels(dev):
    """The long-tag cases of the corpus, each alone and all in one batch: E_PARSE exactly where FromString raises."""
    for kind in (X.REGRESS, X.CLASSIFY):
        wires = [w for _, k, w in X.long_tag_cases() if k == kind]
        for i, w in enumerate(wires):
            check_batch(dev, kind, [w], [i % 128])
        if kind == X.REGRESS:
            check_batch(dev, kind, wires, [i % 16 for i in range(len(wires))])


def test_classify_groups(dev):
    """Classify cases grouped by class count: 127 to 129 and 1000 classes (the first example's body crosses a stage), C = 31 to
    64, labels of 0 to 300 bytes and split UTF-8 characters across the cursor's lines, a late row whose labels differ in their
    last byte."""
    for C_, group in sorted(E.classify_groups().items()):
        names = [g[0] for g in group]
        wires = [g[1] for g in group]
        if "late_row_last_byte" in names:       # same_labels: decided by a row far from the first
            i = names.index("late_row_last_byte")
            for w in (wires[i], wires[names.index("late_row_same")]):
                for rec in (0, 5, 127):
                    check_batch(dev, X.CLASSIFY, [w], [rec])
            keep = [j for j in range(len(wires)) if names[j] not in ("late_row_last_byte", "late_row_same")]
            wires = [wires[j] for j in keep]
        for rec in (0, 3, 64, 127):
            check_batch(dev, X.CLASSIFY, wires, [(rec + 7 * j) % 128 for j in range(len(wires))], host_async=rec == 3)


def test_scan_over_long_runs_of_empty_responses(dev):
    """n = 1023 to 2049 with empty responses first (the first response with rows past 1024) and last; capacities equal to the
    rows used and one less."""
    rng = np.random.default_rng(31)
    for n in (1023, 1024, 1025, 2049):
        lead = min(n - 3, 1030)
        wires = [b""] * lead + [X.random_regression(rng, 5), X.serialize([(1, X.LEN, [])]), X.random_regression(rng, 3)]
        wires += [X.serialize(X.spec_nodes())] * (n - len(wires))
        check_batch(dev, X.REGRESS, wires, [i % 128 for i in range(n)])
        cw = [b""] * lead + [X.random_classification(rng, 4, ["a", "bb"]), X.random_classification(rng, 2, ["a", "bb"])]
        cw += [b""] * (n - len(cw))
        check_batch(dev, X.CLASSIFY, cw, [0] * n)
        for kind, ws, used in ((X.REGRESS, wires, 8), (X.CLASSIFY, cw, 12)):
            last = max(i for i, w in enumerate(ws) if w and _definition(kind, w)[0] == "ok" and len(_definition(kind, w)[1]))
            for cap in (used, used - 1):
                kw = {"values_cap": cap} if kind == X.REGRESS else {"values_cap": used, "labels_cap": cap}
                per, _, batch, vals, refs, *_ = decode_batch(dev, kind, ws, [0] * n, **kw)
                want = N.OK if cap == used else N.E_SIZE
                assert batch[0] == (8 if kind == X.REGRESS else 6) and per[last, 2] == want
                assert batch[3] == want and batch[4] == (-1 if want == N.OK else last)
                assert (vals[used:] == CANARY).all() and (refs[(used if kind == X.CLASSIFY else 0):] == CANARY).all()
                if kind == X.REGRESS:
                    assert (vals[cap:] == CANARY).all()
                else:
                    assert (refs[cap:] == CANARY).all()


def test_group_depth_through_the_kernels_and_python(dev, codec):
    for name, wire, d in E.group_depth_cases():
        per, _, batch, *_ = decode_batch(dev, X.REGRESS, [wire], [0])
        assert per[0, 2] == (N.OK if d <= 16 else N.E_PARSE), name
        calls = codec.example_response_device_calls
        if d >= 100:
            with pytest.raises(DecodeError):
                codec.decode_regression_responses([wire])
            continue
        got = codec.decode_regression_responses([wire])
        assert np.array_equal(_bits(got.values), _bits(X.expected(X.REGRESS, [wire])[0])), name
        assert codec.example_response_device_calls == calls + (1 if d <= 16 else 0), name


def test_python_routes(codec):
    """Every case through Codec.decode_*_responses: the definition's arrays or its exception, by the device route whenever the
    definition decodes."""
    cases = [(c.kind, c.wire) for c in E.regress_grid()] + [(X.REGRESS, w) for _, w in E.emit_cases()]
    cases += [(k, w) for _, k, w in X.long_tag_cases()]
    cases += [(X.CLASSIFY, w) for g in E.classify_groups().values() for _, w in g]
    for kind, wire in cases:
        fn = codec.decode_regression_responses if kind == X.REGRESS else codec.decode_classification_responses
        calls = codec.example_response_device_calls
        try:
            vals, labels, counts = X.expected(kind, [wire])
        except DecodeError:
            with pytest.raises(DecodeError):
                fn([wire])
            continue
        got = fn([wire])
        v = got.values if kind == X.REGRESS else got.scores
        assert np.array_equal(_bits(v), _bits(vals)) and got.counts.tolist() == counts
        if kind == X.CLASSIFY:
            assert got.labels() == labels
        assert codec.example_response_device_calls == calls + 1, "the device route did not finish"


# ---- MultiInference ------------------------------------------------------------------------------------------------------------
def check_multi(dev, kinds, wires, residues):
    lib = dev.lib
    T, n = len(kinds), len(wires)
    img, offs = _place(wires, residues)
    arena = dev.upload(img)
    off = (C.c_uint64 * n)(*offs)
    ln = (C.c_uint64 * n)(*[len(w) for w in wires])
    kv = (C.c_int32 * T)(*kinds)
    mr, mv = (C.c_uint64 * T)(), (C.c_uint64 * T)()
    N.check(lib.b200tfs_multi_inference_response_bound(T, kv, n, ln, mr, mv))
    room = int(mv[0]) + 64
    vs = [dev.upload(np.full(room, CANARY, np.uint32)) for _ in range(T)]
    ls = [dev.upload(np.full(2 * room, CANARY, np.uint32)) for _ in range(T)]
    caps = (C.c_uint64 * T)(*[int(mv[0])] * T)
    lcaps = (C.c_uint64 * T)(*[int(mv[0]) if k == X.CLASSIFY else 0 for k in kinds])
    N.check(lib.b200tfs_decode_multi_inference_responses(dev.ctx, T, kv, arena, n, off, ln, (C.c_void_p * T)(*vs), caps,
                                                         (C.c_void_p * T)(*[l if k == X.CLASSIFY else None for l, k in zip(ls, kinds)]),
                                                         lcaps))
    per, specs, batch = (C.c_int64 * (3 * n * T))(), (N.ModelSpec * (n * T))(), (C.c_int64 * (5 * T))()
    N.check(lib.b200tfs_multi_inference_response_results(dev.ctx, n, T, per, specs, batch))
    per = np.array(per, np.int64).reshape(T, n, 3)
    outcome = []
    for i, w in enumerate(wires):
        try:
            ref = M.expected(kinds, [w])
        except DecodeError:
            assert (per[:, i, 2] == N.E_PARSE).all(), (i, per[:, i, 2])
            outcome.append("parse")
            continue
        except ValueError:
            assert N.E_PARSE not in per[:, i, 2] and N.E_SHAPE in per[:, i, 2], i
            outcome.append("shape")
            continue
        assert (per[:, i, 2] == N.OK).all(), (i, per[:, i, 2])
        for t, (rv, rl, counts, rspecs) in enumerate(ref):
            assert per[t, i, 1] == counts[0] and _spec_ok(w, specs[t * n + i], rspecs[0]), (i, t)
        outcome.append(("ok", ref))
    for t, k in enumerate(kinds):
        total = int(batch[5 * t])
        C_ = int(batch[5 * t + 1]) if k == X.CLASSIFY else 1
        vals = dev.download(vs[t], 4 * room, np.uint32)
        refs = dev.download(ls[t], 8 * room, np.uint32).reshape(-1, 2)
        assert (vals[total * C_:] == CANARY).all() and (refs[total * C_:] == CANARY).all()
        for i, o in enumerate(outcome):
            if o in ("parse", "shape"):
                continue
            rv, rl = o[1][t][0], o[1][t][1]
            r0, rows = int(per[t, i, 0]), int(per[t, i, 1])
            assert np.array_equal(vals[r0 * C_: (r0 + rows) * C_], _bits(rv).ravel()), (i, t)
            if k == X.CLASSIFY:
                got = [[img[offs[i] + int(refs[(r0 + j) * C_ + c, 0]): offs[i] + int(refs[(r0 + j) * C_ + c, 0]) + int(refs[(r0 + j) * C_ + c, 1])]
                        .tobytes() for c in range(C_)] for j in range(rows)]
                assert got == [[lab.encode() for lab in r] for r in rl], (i, t)
    return outcome


def test_multi_inference_edges(dev, codec):
    """The window, stage and tag cases inside a task's member body, 1 to 4 tasks, the oneof and repeated-member cases: each
    alone at two residues, batched by task kinds, and through the Python route."""
    from min_tfs_client.requests import CLASSIFY_METHOD_NAME, REGRESS_METHOD_NAME

    by_kinds = {}
    for c in E.multi_cases():
        by_kinds.setdefault(tuple(c.kind), []).append(c)
    seen = {}
    for kinds, cases in by_kinds.items():
        for rec in (0, 9):
            for o in check_multi(dev, list(kinds), [c.wire for c in cases], [(rec + 5 * j) % 128 for j in range(len(cases))]):
                key = o if isinstance(o, str) else "ok"
                seen[key] = seen.get(key, 0) + 1
        methods = [CLASSIFY_METHOD_NAME if k == X.CLASSIFY else REGRESS_METHOD_NAME for k in kinds]
        for c in cases:
            calls = codec.multi_inference_device_calls
            try:
                ref = M.expected(list(kinds), [c.wire])
            except (DecodeError, ValueError) as e:
                with pytest.raises(type(e)):
                    codec.decode_multi_inference_responses([c.wire], methods)
                continue
            got = codec.decode_multi_inference_responses([c.wire], methods)
            for g, (rv, rl, counts, _), k in zip(got, ref, kinds):
                v = g.values if k == X.REGRESS else g.scores
                assert np.array_equal(_bits(v), _bits(rv)) and g.counts.tolist() == counts, c.name
            assert codec.multi_inference_device_calls == calls + 1, c.name
    print("multi outcomes:", seen)
    assert seen.get("ok", 0) > 80 and seen.get("parse", 0) > 10
