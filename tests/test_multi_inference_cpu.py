"""MultiInference without a GPU: the inference.proto schema module, the closed-form size of MultiInferenceRequests against the
protobuf runtime, the refusals of the *_example_tasks* entry points (checked before the context is looked at), and the response
walk (csrc/multi_walk.h) compiled for the host against the definition on server-written responses, every edge case and a seeded
mutant corpus.  The GPU test runs the same corpus through the kernels."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
from google.protobuf import descriptor as D
from google.protobuf.message import DecodeError

import multi_inference_corpus as M
from min_tfs_client import _native as N
from min_tfs_client.codec import _example_columns
from min_tfs_client.requests import CLASSIFY_METHOD_NAME, REGRESS_METHOD_NAME, make_multi_inference_request
from tensorflow_serving.apis import inference_pb2

HERE = os.path.dirname(os.path.abspath(__file__))
F = D.FieldDescriptor


# ---- schema ----------------------------------------------------------------------------------------------------------------
SCHEMA = {   # message: [(name, number, type, label, oneof)] as TF Serving's inference.proto has them
    "InferenceTask": [("model_spec", 1, F.TYPE_MESSAGE, F.LABEL_OPTIONAL, None), ("method_name", 2, F.TYPE_STRING, F.LABEL_OPTIONAL, None)],
    "InferenceResult": [("model_spec", 1, F.TYPE_MESSAGE, F.LABEL_OPTIONAL, None),
                        ("classification_result", 2, F.TYPE_MESSAGE, F.LABEL_OPTIONAL, "result"),
                        ("regression_result", 3, F.TYPE_MESSAGE, F.LABEL_OPTIONAL, "result")],
    "MultiInferenceRequest": [("tasks", 1, F.TYPE_MESSAGE, F.LABEL_REPEATED, None), ("input", 2, F.TYPE_MESSAGE, F.LABEL_OPTIONAL, None)],
    "MultiInferenceResponse": [("results", 1, F.TYPE_MESSAGE, F.LABEL_REPEATED, None)],
}
TYPES = {("InferenceTask", "model_spec"): "tensorflow.serving.ModelSpec", ("InferenceResult", "model_spec"): "tensorflow.serving.ModelSpec",
         ("InferenceResult", "classification_result"): "tensorflow.serving.ClassificationResult",
         ("InferenceResult", "regression_result"): "tensorflow.serving.RegressionResult",
         ("MultiInferenceRequest", "tasks"): "tensorflow.serving.InferenceTask", ("MultiInferenceRequest", "input"): "tensorflow.serving.Input",
         ("MultiInferenceResponse", "results"): "tensorflow.serving.InferenceResult"}


@pytest.mark.parametrize("msg", sorted(SCHEMA))
def test_schema_fields(msg):
    d = getattr(inference_pb2, msg).DESCRIPTOR
    assert d.full_name == "tensorflow.serving." + msg and d.file.package == "tensorflow.serving"
    got = [(f.name, f.number, f.type, f.label, f.containing_oneof.name if f.containing_oneof else None) for f in d.fields]
    assert sorted(got) == sorted(SCHEMA[msg])
    for f in d.fields:
        if f.type == F.TYPE_MESSAGE:
            assert f.message_type.full_name == TYPES[(msg, f.name)]


# ---- request sizes and refusals --------------------------------------------------------------------------------------------
def _structs(d, ctx, name="m", version=2, grpc_frame=False):
    n, preps = _example_columns(d)
    feats = (N.Feature * max(len(preps), 1))(*[p[0] for p in preps])
    nb = name.encode()
    req = N.ExampleRequest(model_name=nb, model_name_len=len(nb), has_version=int(version is not None), order=N.ORDER_UPB,
                           version=version or 0, n_examples=n, n_features=len(preps), flags=N.RF_GRPC_FRAME if grpc_frame else 0,
                           features=feats)
    keep = [preps, feats, nb]
    cx = None
    if ctx is not None:
        _, cpreps = _example_columns(ctx, context=True)
        cfeats = (N.Feature * max(len(cpreps), 1))(*[p[0] for p in cpreps])
        cx = N.ExampleContext(features=cfeats, n_features=len(cpreps), present=1)
        keep += [cpreps, cfeats]
    return req, cx, keep


def _tasks(tasks):
    sigs = [s.encode() for s, _ in tasks]
    arr = (N.InferenceTask * max(len(tasks), 1))(*[N.InferenceTask(signature_name=s, signature_len=len(s),
                                                                     method=N.RESP_CLASSIFY if m == CLASSIFY_METHOD_NAME else N.RESP_REGRESS)
                                                     for s, (_, m) in zip(sigs, tasks)])
    return N.ExampleTasks(tasks=C.addressof(arr), n_tasks=len(tasks)), (arr, sigs)


SIGS = ["", "serving_default", "ünïcødé-€", "s" * 130]
CASES = [(t, sig, ver, ctx) for t in (1, 2, 3, 5) for sig in SIGS for ver in (None, 0, 2 ** 40 + 3) for ctx in (False, True)]


@pytest.mark.parametrize("n_tasks,sig,version,ctx", CASES)
def test_request_size_matches_protobuf(n_tasks, sig, version, ctx):
    rng = np.random.default_rng(n_tasks)
    d = {"x": rng.standard_normal((3, 4)).astype(np.float32), "w": np.float32(0.5)}
    cd = {"q": rng.standard_normal(5).astype(np.float32)} if ctx else None
    tasks = [(sig if k % 2 == 0 else "", CLASSIFY_METHOD_NAME if k % 3 != 1 else REGRESS_METHOD_NAME) for k in range(n_tasks)]
    want = len(make_multi_inference_request("model", version, tasks, d, cd).SerializeToString(deterministic=True))
    for frame in (False, True):
        req, cx, keep = _structs(d, cd, "model", version, frame)
        tk, keep2 = _tasks(tasks)
        out = C.c_uint64()
        N.check(N.load().b200tfs_example_tasks_request_size(C.byref(req), None, C.byref(cx) if cx else None, C.byref(tk), C.byref(out)))
        assert out.value == want + (5 if frame else 0)


def test_no_tasks_is_the_request_without_tasks():
    d = {"x": np.ones((2, 3), np.float32)}
    req, _, keep = _structs(d, None)
    tk = N.ExampleTasks(tasks=None, n_tasks=0)
    a, b = C.c_uint64(), C.c_uint64()
    N.check(N.load().b200tfs_example_tasks_request_size(C.byref(req), None, None, C.byref(tk), C.byref(a)))
    N.check(N.load().b200tfs_example_context_request_size(C.byref(req), None, None, C.byref(b)))
    assert a.value == b.value


def _rcs(req, tg, tk):
    """request size, arena size, _host and _async with no device context: their argument checks"""
    lib = N.load()
    out = C.c_uint64()
    off, ln = (C.c_uint64 * 1)(), (C.c_uint64 * 1)()
    buf = C.create_string_buffer(256)
    t = C.byref(tg) if tg is not None else None
    return [lib.b200tfs_example_tasks_request_size(C.byref(req), t, None, C.byref(tk), C.byref(out)),
            lib.b200tfs_example_tasks_arena_size(1, C.byref(req), None, t, None, None, C.byref(tk), C.byref(out)),
            lib.b200tfs_encode_example_tasks_host(None, 1, C.byref(req), None, None, t, None, None, C.byref(tk), buf, 16, off, ln),
            lib.b200tfs_encode_example_tasks_async(None, 1, C.byref(req), None, None, t, None, None, C.byref(tk), buf, 16)]


def test_refusals():
    req, _, keep = _structs({"x": np.ones((2, 3), np.float32)}, None)
    good, keep2 = _tasks([("s", CLASSIFY_METHOD_NAME)])
    arr = keep2[0]
    bad = [N.ExampleTasks(tasks=C.addressof(arr), n_tasks=-1), N.ExampleTasks(tasks=None, n_tasks=1)]
    for method in (0, 3, -1):
        a = (N.InferenceTask * 1)(N.InferenceTask(signature_name=b"s", signature_len=1, method=method))
        keep.append(a)
        bad.append(N.ExampleTasks(tasks=C.addressof(a), n_tasks=1))
    for sig, ln in ((b"s", -1), (None, 3)):
        a = (N.InferenceTask * 1)(N.InferenceTask(signature_name=sig, signature_len=ln, method=N.RESP_REGRESS))
        keep.append(a)
        bad.append(N.ExampleTasks(tasks=C.addressof(a), n_tasks=1))
    for tk in bad:
        assert _rcs(req, None, tk) == [N.E_ARG] * 4
    for kind in (N.EXAMPLES_PREDICT_STRING,):
        tg = N.ExampleTarget(kind=kind, key=b"k", key_len=1)
        assert _rcs(req, tg, good) == [N.E_ARG] * 4
    # the same arguments without a device context get as far as the context (E_ARG for it), the sizes succeed
    rcs = _rcs(req, N.ExampleTarget(kind=N.EXAMPLES_LIST, key=None, key_len=0), good)
    assert rcs[:2] == [N.OK, N.OK]


def test_python_refusals():
    with pytest.raises(ValueError):
        make_multi_inference_request("m", None, [], {"x": np.ones((1, 1), np.float32)})
    with pytest.raises(ValueError):
        make_multi_inference_request("m", None, [("s", "tensorflow/serving/predict")], {"x": np.ones((1, 1), np.float32)})


# ---- the response walk on the host -----------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    cxx = os.environ.get("CXX") or shutil.which("g++") or "c++"
    so = str(tmp_path_factory.mktemp("mw") / "libmulti_walk_host.so")
    subprocess.run([cxx, "-O2", "-std=c++17", "-fPIC", "-Wall", "-Wno-unknown-pragmas", "-shared", "-o", so,
                    os.path.join(HERE, "native", "multi_inference_walk_host.cpp")], check=True)
    L = C.CDLL(so)
    L.mw_decode.restype = None
    L.mw_decode.argtypes = [C.c_int, C.POINTER(C.c_int), C.c_char_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint64,
                            C.POINTER(C.c_int), C.POINTER(C.c_uint64), C.POINTER(C.c_int64), C.POINTER(N.ModelSpec)]
    L.mw_row_bound.restype = C.c_uint64
    L.mw_row_bound.argtypes = [C.c_uint64]
    return L


def walk(lib, kinds, wire):
    T = len(kinds)
    cap = max(len(wire) // 2, 1)
    vals = np.zeros((T, cap), np.float32)
    refs = (N.LabelRef * (T * cap))()
    st, rows, ncls, specs = (C.c_int * T)(), (C.c_uint64 * T)(), (C.c_int64 * T)(), (N.ModelSpec * T)()
    lib.mw_decode(T, (C.c_int * T)(*kinds), wire, len(wire), vals.ctypes.data, C.addressof(refs), cap, st, rows, ncls, specs)
    out = []
    for t, k in enumerate(kinds):
        r, c = rows[t], ncls[t]
        if k == M.REGRESS or st[t] != N.OK:
            out.append((st[t], vals[t, :r], None, r, specs[t]))
            continue
        lab = [[wire[refs[t * cap + i * c + j].off: refs[t * cap + i * c + j].off + refs[t * cap + i * c + j].len].decode() for j in range(c)]
               for i in range(r)]
        out.append((st[t], vals[t, : r * c].reshape(r, c), lab, r, specs[t]))
    return out


def check(lib, kinds, wire, what=""):
    got = walk(lib, kinds, wire)
    sts = [g[0] for g in got]
    try:
        ref = M.expected(kinds, [wire])
    except DecodeError:
        assert N.E_PARSE in sts, (what, sts, wire.hex())
        return "parse"
    except ValueError:
        assert N.E_PARSE not in sts and N.E_SHAPE in sts, (what, sts, wire.hex())
        return "shape"
    assert sts == [N.OK] * len(kinds), (what, sts, wire.hex())
    for (st, vals, lab, rows, spec), (rv, rl, counts, rspecs) in zip(got, ref):
        assert rows == counts[0], what
        assert vals.view(np.uint32).tolist() == rv.view(np.uint32).tolist(), (what, wire.hex())
        assert lab == rl, what
        ms = rspecs[0]
        text = lambda off, n: wire[off: off + n].decode()   # noqa: E731
        assert text(spec.name_off, spec.name_len) == ms.name and text(spec.signature_off, spec.signature_len) == ms.signature_name
        assert bool(spec.has_version) == ms.HasField("version") and (not spec.has_version or spec.version == ms.version.value)
        assert text(spec.label_off, spec.label_len) == ms.version_label
    return "ok"


def test_server_written_responses(lib):
    rng = np.random.default_rng(1)
    for kinds in ([M.CLASSIFY], [M.REGRESS], [M.CLASSIFY, M.REGRESS], [M.REGRESS, M.CLASSIFY, M.CLASSIFY, M.REGRESS]):
        for n in (0, 1, 7, 300):
            assert check(lib, kinds, M.random_response(rng, kinds, n)) == "ok"
            assert check(lib, kinds, M.random_response(rng, kinds, n, labels=lambda i: [f"top{i}", "ü", ""])) == "ok"


@pytest.mark.parametrize("name,kinds,wire", M.edge_cases(), ids=[c[0] for c in M.edge_cases()])
def test_edge_cases_match_the_definition(lib, name, kinds, wire):
    check(lib, kinds, wire, name)


def test_edge_case_outcomes_are_the_expected_ones(lib):
    got = {name: check(lib, kinds, wire, name) for name, kinds, wire in M.edge_cases()}
    for name in ("plain", "oneof_2_3", "oneof_3_2", "oneof_2_3_2", "member_merge", "spec_merge", "unknown_everywhere",
                 "member_wrong_wire_type", "results_wrong_wire_type", "empty_bodies", "snan"):
        assert got[name] == "ok", name
    for name in ("oneof_2_3_2_as_regress", "zero_results", "fewer_results", "more_results", "wrong_case", "empty_result",
                 "empty_result_spec_only", "ragged_classes"):
        assert got[name] == "shape", name
    for name in ("cleared_bad_utf8", "cleared_truncated_value", "past_tasks_bad_utf8", "wrong_case_bad_utf8", "decoded_bad_utf8",
                 "spec_bad_utf8", "tag_zero", "length_past_end", "open_group"):
        assert got[name] == "parse", name
    wire = dict((c[0], c[2]) for c in M.edge_cases())["oneof_2_3_2"]
    assert walk(lib, [M.CLASSIFY], wire)[0][2] == [["b"]]      # the last classification_result alone
    wire = dict((c[0], c[2]) for c in M.edge_cases())["member_merge"]
    assert walk(lib, [M.REGRESS, M.CLASSIFY], wire)[0][1].tolist() == [1.0, 2.0, 3.0]


def test_mutant_corpus_matches_the_definition(lib):
    outcomes = {"ok": 0, "parse": 0, "shape": 0}
    for i, (kinds, wire) in enumerate(M.mutants()):
        outcomes[check(lib, kinds, wire, f"mutant {i}")] += 1
    assert outcomes["ok"] > 50 and outcomes["parse"] > 100 and outcomes["shape"] > 10, outcomes
