"""The Classify / Regress response walk (csrc/example_walk.h), compiled for the host, against the protobuf runtime.

CPU only: the walk composed the way the kernels compose it (tests/native/example_walk_host.cpp) must agree with
ClassificationResponse.FromString / RegressionResponse.FromString on server-written responses, on every edge case the runtime's
behaviour pins, and on a seeded mutant corpus: DecodeError exactly where the walk says B200TFS_E_PARSE, bit-equal values and
equal labels everywhere else.  The GPU test runs the same corpus through the kernels.
"""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

import example_response_corpus as X
from min_tfs_client import _native as N

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    cxx = os.environ.get("CXX") or shutil.which("g++") or "c++"
    so = str(tmp_path_factory.mktemp("xw") / "libexample_walk_host.so")
    subprocess.run([cxx, "-O2", "-std=c++17", "-fPIC", "-Wall", "-Wno-unknown-pragmas", "-shared", "-o", so,
                    os.path.join(HERE, "native", "example_walk_host.cpp")], check=True)
    L = C.CDLL(so)
    L.xw_decode.restype = C.c_int
    L.xw_decode.argtypes = [C.c_int, C.c_char_p, C.c_uint64, C.c_int64, C.c_void_p, C.c_void_p, C.c_uint64,
                            C.POINTER(C.c_uint64), C.POINTER(C.c_int64), C.POINTER(N.ModelSpec)]
    L.xw_row_bound.restype = C.c_uint64
    L.xw_row_bound.argtypes = [C.c_uint64]
    return L


def walk(lib, kind, wire, C_in=-1):
    """(status, values or scores, labels, rows, n_classes, spec)"""
    cap = max(len(wire) // 2, 1)      # rows, and rows * C of a response that decodes
    vals = np.zeros(cap, np.float32)
    refs = (N.LabelRef * cap)()
    rows, ncls, spec = C.c_uint64(), C.c_int64(), N.ModelSpec()
    st = lib.xw_decode(kind, wire, len(wire), C_in, vals.ctypes.data, C.addressof(refs), cap, C.byref(rows), C.byref(ncls), C.byref(spec))
    r, c = rows.value, ncls.value
    if kind == X.REGRESS or st != N.OK:
        return st, vals[:r], None, r, c, spec
    labels = [[wire[refs[i * c + k].off: refs[i * c + k].off + refs[i * c + k].len].decode("utf-8") for k in range(c)] for i in range(r)]
    return st, vals[: r * c].reshape(r, c), labels, r, c, spec


def check(lib, kind, wire, what=""):
    from google.protobuf.message import DecodeError

    st, vals, labels, rows, ncls, spec = walk(lib, kind, wire)
    assert st in (N.OK, N.E_PARSE, N.E_SHAPE), (what, st)
    try:
        ref_vals, ref_labels, counts = X.expected(kind, [wire])
    except DecodeError:
        assert st == N.E_PARSE, (what, wire.hex())
        return "parse"
    except ValueError:
        assert st == N.E_SHAPE, (what, wire.hex())
        return "shape"
    assert st == N.OK, (what, st, wire.hex())
    assert rows == counts[0], what
    assert vals.view(np.uint32).tolist() == ref_vals.view(np.uint32).tolist(), (what, wire.hex())
    if kind == X.CLASSIFY:
        assert labels == ref_labels, what
    from tensorflow_serving.apis.regression_pb2 import RegressionResponse

    ms = RegressionResponse.FromString(wire).model_spec if kind == X.REGRESS else None
    if ms is not None:
        text = lambda off, n: wire[off: off + n].decode("utf-8")   # noqa: E731
        assert text(spec.name_off, spec.name_len) == ms.name and text(spec.signature_off, spec.signature_len) == ms.signature_name
        assert bool(spec.has_version) == ms.HasField("version") and (not spec.has_version or spec.version == ms.version.value)
        assert text(spec.label_off, spec.label_len) == ms.version_label
    return "ok"


def test_server_written_responses(lib):
    rng = np.random.default_rng(1)
    for n in (0, 1, 7, 300):
        assert check(lib, X.REGRESS, X.random_regression(rng, n)) == "ok"
        assert check(lib, X.CLASSIFY, X.random_classification(rng, n, ["0", "1"])) == "ok"
        assert check(lib, X.CLASSIFY, X.random_classification(rng, n, lambda i: [f"top{i}", "ü", ""])) == "ok"


@pytest.mark.parametrize("name,kind,wire", X.edge_cases(), ids=[c[0] for c in X.edge_cases()])
def test_edge_cases_match_the_runtime(lib, name, kind, wire):
    check(lib, kind, wire, name)


def test_edge_case_outcomes_are_the_expected_ones(lib):
    """The corpus exercises what it claims to: decodes, parse errors and ragged class counts all occur."""
    got = {name: check(lib, kind, wire, name) for name, kind, wire in X.edge_cases()}
    assert got["regress_repeated_result"] == got["regress_unknown_everywhere"] == got["classify_utf8"] == "ok"
    assert got["classify_ragged"] == "shape"
    for name in ("classify_bad_utf8", "classify_surrogate", "spec_bad_utf8", "tag_zero", "wire_type_6", "mismatched_group",
                 "varint_11_bytes", "length_past_end", "truncated_value"):
        assert got[name] == "parse", name
    st, vals, *_ = walk(lib, X.REGRESS, dict((c[0], c[2]) for c in X.edge_cases())["regress_snan"])
    assert vals.view(np.uint32).tolist() == [0x7FC00001]


def test_mutant_corpus_matches_the_runtime(lib):
    outcomes = {"ok": 0, "parse": 0, "shape": 0}
    for i, (kind, wire) in enumerate(X.mutants()):
        outcomes[check(lib, kind, wire, f"mutant {i}")] += 1
    assert outcomes["ok"] > 100 and outcomes["parse"] > 100, outcomes


def test_bound_covers_rows_and_classes(lib):
    rng = np.random.default_rng(5)
    for _ in range(200):
        n = int(rng.integers(0, 40))
        if rng.integers(2):
            wire = X.random_regression(rng, n)
            st, _, _, rows, _, _ = walk(lib, X.REGRESS, wire)
            assert rows <= lib.xw_row_bound(len(wire))
        else:
            c = int(rng.integers(0, 6))
            wire = X.random_classification(rng, n, [""] * c)   # the smallest classes there are
            st, _, _, rows, ncls, _ = walk(lib, X.CLASSIFY, wire)
            assert rows <= lib.xw_row_bound(len(wire)) and ncls <= lib.xw_row_bound(len(wire))
            assert rows * ncls <= lib.xw_row_bound(len(wire))
        assert st == N.OK
