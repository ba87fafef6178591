"""The edges of the Classify / Regress / MultiInference warp entry finder, without a GPU: the restatement of its schedule
(tests/xr_edges.py) and the host walk (csrc/example_walk.h, csrc/multi_walk.h) against FromString on every case of the grid, a
coverage assertion that every edge of the grid is reached, and the tag and group-depth rules.  The GPU test runs the same grid
through the kernels."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
from google.protobuf.message import DecodeError

import example_response_corpus as X
import multi_inference_corpus as M
import xr_edges as E
from min_tfs_client import _native as N
from test_example_response_walk_cpu import check as walk_check
from test_example_response_walk_cpu import walk
from test_multi_inference_cpu import check as mi_check

HERE = os.path.dirname(os.path.abspath(__file__))
RESIDUES = list(range(16)) + [17, 50, 63, 64, 100, 127]      # of the record's device address: mod 16 (staging), mod 128 (lines)


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    cxx = os.environ.get("CXX") or shutil.which("g++") or "c++"
    so = str(tmp_path_factory.mktemp("xe") / "libexample_walk_host.so")
    subprocess.run([cxx, "-O2", "-std=c++17", "-fPIC", "-Wall", "-Wno-unknown-pragmas", "-shared", "-o", so,
                    os.path.join(HERE, "native", "example_walk_host.cpp")], check=True)
    L = C.CDLL(so)
    L.xw_decode.restype = C.c_int
    L.xw_decode.argtypes = [C.c_int, C.c_char_p, C.c_uint64, C.c_int64, C.c_void_p, C.c_void_p, C.c_uint64,
                            C.POINTER(C.c_uint64), C.POINTER(C.c_int64), C.POINTER(N.ModelSpec)]
    return L


def restated(kind, wire):
    """(values or scores rows, labels) the restatement's entries give, parsed entry by entry; DecodeError when it errs"""
    from tensorflow_serving.apis.classification_pb2 import Classifications
    from tensorflow_serving.apis.regression_pb2 import Regression

    sch = E.response_schedules(wire)
    if sch is None or any(S.err for S in sch):
        raise DecodeError("the finder stops on a malformed field")
    ents = [wire[o: o + n] for S in sch for o, n in S.entries]
    if kind == X.REGRESS:
        return np.array([Regression.FromString(e).value for e in ents], np.float32), None
    rows = [[(c.label, c.score) for c in Classifications.FromString(e).classes] for e in ents]
    return [[s for _, s in r] for r in rows], [[lab for lab, _ in r] for r in rows]


def _bits(a):
    return np.asarray(a, np.float32).view(np.uint32).tolist()


def agree(lib, kind, wire, name):
    """the restatement and the host walk against FromString; the outcome"""
    try:
        want = X.expected(kind, [wire])
    except DecodeError:
        with pytest.raises(DecodeError):
            restated(kind, wire)
        assert walk_check(lib, kind, wire, name) == "parse", name
        return "parse"
    got, labels = restated(kind, wire)
    if kind == X.REGRESS:
        assert _bits(got) == _bits(want[0]), name
    else:
        assert [_bits(r) for r in got] == [_bits(r) for r in want[0]] and labels == want[1], name
    assert walk_check(lib, kind, wire, name) == "ok", name
    return "ok"


def grid(rec=0):
    cases = E.regress_grid(rec)
    for C_, group in E.classify_groups().items():
        cases += [E.Case(name, X.CLASSIFY, w, rec) for name, w in group]
    cases += [E.Case(name, X.REGRESS, w, rec) for name, w in E.emit_cases()]
    return cases


def wanted_edges():
    """every edge the grid is there to reach"""
    want = set()
    for kind, _ in E.body_fields():
        want |= {("start", kind, k) for k in (253, 254, 255, 256)} | {("end", kind, e) for e in (255, 256, 257)}
    want |= {("chain", n) for n in (126, 127, 128)} | {("chain", n, "odd") for n in (126, 127)} | {("chain", 128, "ends_at_L")}
    want |= {("stage", "need_eq"), ("stage", "need_eq+1"), ("group_skip", ">4K"), ("group_skip", ">8K"), ("result2_later_stage",)}
    want |= {("restage_rec16", r) for r in range(16)} | {("restage_rec128", r) for r in RESIDUES}
    want |= {("tail", w) for w in (2, 7, 9, 11, 15)}
    want |= {("err", kind, where) for kind, _ in E.bad_fields() for where in ("window0", "pos255", "stage2")}
    want |= {("classes", C_, "restaged") for C_ in (127, 128, 129, 1000)}
    return want


def test_restatement_and_host_walk_agree_with_the_runtime_on_the_grid(lib):
    outcomes = {"ok": 0, "parse": 0}
    for c in grid():
        outcomes[agree(lib, c.kind, c.wire, c.name)] += 1
    print("grid outcomes:", outcomes)
    assert outcomes["ok"] > 500 and outcomes["parse"] >= 21


def test_every_edge_of_the_grid_is_reached():
    counts = {}
    for rec in RESIDUES:
        for c in grid(rec):
            for e in E.edges(c, rec):
                counts[e] = counts.get(e, 0) + 1
    want = wanted_edges()
    missing = sorted(want - set(counts), key=str)
    by_family = {}
    for e, n in counts.items():
        by_family[e[0]] = by_family.get(e[0], 0) + n
    print("edge families reached:", ", ".join(f"{k} {v}" for k, v in sorted(by_family.items())))
    print(f"{len(want) - len(missing)}/{len(want)} wanted edges reached")
    assert not missing, missing


@pytest.fixture(scope="module")
def mi_lib(tmp_path_factory):
    cxx = os.environ.get("CXX") or shutil.which("g++") or "c++"
    so = str(tmp_path_factory.mktemp("me") / "libmulti_walk_host.so")
    subprocess.run([cxx, "-O2", "-std=c++17", "-fPIC", "-Wall", "-Wno-unknown-pragmas", "-shared", "-o", so,
                    os.path.join(HERE, "native", "multi_inference_walk_host.cpp")], check=True)
    L = C.CDLL(so)
    L.mw_decode.restype = None
    L.mw_decode.argtypes = [C.c_int, C.POINTER(C.c_int), C.c_char_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint64,
                            C.POINTER(C.c_int), C.POINTER(C.c_uint64), C.POINTER(C.c_int64), C.POINTER(N.ModelSpec)]
    return L


def test_multi_inference_grid_matches_the_runtime(mi_lib):
    """MultiInference cases: the host walk against the definition, and the restatement over every member body the finder walks
    against FromString's entries."""
    from tensorflow_serving.apis.inference_pb2 import MultiInferenceResponse

    outcomes = {}
    for c in E.multi_cases():
        got = mi_check(mi_lib, c.kind, c.wire, c.name)
        outcomes[got] = outcomes.get(got, 0) + 1
        if got != "ok":
            continue
        bodies = E.member_bodies(c.wire, c.kind)
        ents = [c.wire[o: o + n] for lo, hi in bodies for o, n in E.warp_entries(c.wire, lo, hi).entries]
        m = MultiInferenceResponse.FromString(c.wire)
        want = [r.regression_result.regressions if k == X.REGRESS else r.classification_result.classifications
                for r, k in zip(m.results, c.kind)]
        assert len(ents) == sum(len(w) for w in want), c.name
    print("multi outcomes:", outcomes)
    assert outcomes.get("ok", 0) > 40 and outcomes.get("parse", 0) >= 9, outcomes


# ---- the tag rule and the group-depth limit ------------------------------------------------------------------------------------
def test_long_tags_are_refused_like_the_runtime(lib):
    """A tag of 6 to 10 bytes is malformed wherever it stands; one of 5 bytes is read when its value fits 32 bits."""
    seen = {}
    for name, kind, wire in X.long_tag_cases():
        got = agree(lib, kind, wire, name)
        seen[name] = got
    for n in range(6, 11):
        for where in ("result", "entry", "value", "unknown", "unknown_body", "group_member", "class", "label"):
            assert seen[f"{where}_tag_{n}_bytes"] == "parse", (where, n)
    for where in ("result", "entry", "value", "unknown", "class"):
        assert seen[f"{where}_tag_5_bytes"] == "ok", where
    assert seen["unknown_tag_5th_byte_0f"] == "ok" and seen["unknown_tag_5th_byte_10"] == "parse"


def test_group_depth_limit(lib):
    """Unknown groups nested up to 16 deep are skipped; deeper ones are B200TFS_E_PARSE in the walk (and the finder), while the
    runtime accepts them up to its recursion limit (99 inside a result body) - the Python layer gives the runtime's answer by
    the host route."""
    for name, wire, d in E.group_depth_cases():
        st = walk(lib, X.REGRESS, wire)[0]
        assert st == (N.OK if d <= 16 else N.E_PARSE), name
        sch = E.response_schedules(wire)
        assert any(S.err for S in sch) == (d > 16), name
        try:
            X.expected(X.REGRESS, [wire])
            ok = True
        except DecodeError:
            ok = False
        assert ok == (d < 100), name
