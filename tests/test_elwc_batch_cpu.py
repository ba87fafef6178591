"""Predict requests carrying a batch of ExampleListWithContexts (one per query): elwcs_from_input_dict and
make_predict_elwcs_request against hand-built protobuf messages, and the C ABI's host arithmetic (b200tfs_example_lists_
request_size / _arena_size, no kernel): every refusal, and the arena bound against the protobuf size."""
import ctypes as C

import numpy as np
import pytest

from min_tfs_client import _native as N
from min_tfs_client.codec import BytesColumn, RaggedColumn, _example_columns
from min_tfs_client.requests import elwcs_from_input_dict, make_predict_elwcs_request
from tensorflow.core.example.example_pb2 import Example
from tensorflow_serving.apis.input_pb2 import ExampleListWithContext
from tensorflow_serving.apis.predict_pb2 import PredictRequest


def _example(feats):
    ex = Example()
    for k, (kind, vals) in feats.items():
        getattr(ex.features.feature[k], kind).value.extend(vals)
    return ex


def _hand(contexts, lists):
    """ELWCs from explicit per-query contexts and example lists of {key: (kind, values)}"""
    out = []
    for ctx, exs in zip(contexts, lists):
        e = ExampleListWithContext()
        e.examples.extend(_example(f) for f in exs)
        e.context.SetInParent()
        e.context.CopyFrom(_example(ctx))
        out.append(e)
    return out


def _same(got, want):
    assert [g.SerializeToString(deterministic=True) for g in got] == [w.SerializeToString(deterministic=True) for w in want]


@pytest.mark.parametrize("sizes", [[2, 1], [0, 3], [2, 0, 1], [3, 0], [0, 0, 0], [1]])
def test_elwcs_dense_and_broadcast_against_hand_built(sizes):
    n, Q = sum(sizes), len(sizes)
    x = np.arange(2 * n, dtype=np.float32).reshape(n, 2)
    ids = np.arange(n, dtype=np.int64) * 7 - 3
    user = np.arange(Q * 3, dtype=np.float64).reshape(Q, 3) / 4
    got = elwcs_from_input_dict({"user": user, "k": np.int32(5)}, {"x": x, "ids": ids, "c": np.float16(1.5)}, sizes)
    contexts = [{"user": ("float_list", user[q].tolist()), "k": ("int64_list", [5])} for q in range(Q)]
    lists, s = [], 0
    for m in sizes:
        lists.append([{"x": ("float_list", x[j].tolist()), "ids": ("int64_list", [int(ids[j])]), "c": ("float_list", [1.5])}
                      for j in range(s, s + m)])
        s += m
    _same(got, _hand(contexts, lists))


def test_elwcs_empty_context_and_q0():
    got = elwcs_from_input_dict({}, {"x": np.ones((3, 1), np.float32)}, np.array([1, 2], np.uint8))
    assert [e.SerializeToString(deterministic=True)[-2:] for e in got] == [b"\x12\x00"] * 2
    assert elwcs_from_input_dict({}, {}, []) == []
    req = make_predict_elwcs_request("m", 1, {}, {}, np.zeros(0, np.int64), "q")
    t = req.inputs["q"]
    assert list(t.tensor_shape.dim)[0].size == 0 and len(t.string_val) == 0


def test_elwcs_ragged_and_bytes_contexts():
    Q = 3
    toks = RaggedColumn(np.arange(Q * 4, dtype=np.int64).reshape(Q, 4), np.array([2, 0, 4]))
    text = BytesColumn.from_array(np.array([b"a", b"", b"\x00z"], object).astype("S2"))
    words = RaggedColumn(BytesColumn.from_array(np.array([[b"p", b"q"], [b"r", b"s"], [b"t", b"u"]], "S1")), np.array([1, 2, 0]))
    got = elwcs_from_input_dict({"toks": toks, "text": text, "words": words}, {"x": np.zeros((2, 1), np.float32)}, [1, 0, 1])
    contexts = [{"toks": ("int64_list", [0, 1]), "text": ("bytes_list", [b"a"]), "words": ("bytes_list", [b"p"])},
                {"toks": ("int64_list", []), "text": ("bytes_list", [b""]), "words": ("bytes_list", [b"r", b"s"])},
                {"toks": ("int64_list", [8, 9, 10, 11]), "text": ("bytes_list", [b"\x00z"]), "words": ("bytes_list", [])}]
    lists = [[{"x": ("float_list", [0.0])}], [], [{"x": ("float_list", [0.0])}]]
    _same(got, _hand(contexts, lists))


def test_elwcs_value_errors():
    with pytest.raises(ValueError, match="rows"):
        elwcs_from_input_dict({}, {"x": np.zeros((3, 1))}, [1, 1])
    with pytest.raises(ValueError, match="rows"):
        elwcs_from_input_dict({"u": np.zeros(3)}, {"x": np.zeros((2, 1))}, [1, 1])
    with pytest.raises(ValueError, match=">= 0"):
        elwcs_from_input_dict({}, {"x": np.zeros((0, 1))}, [1, -1])
    with pytest.raises(ValueError):
        elwcs_from_input_dict({}, {}, [[1]])


def test_make_predict_elwcs_request_and_spec_fields():
    user = np.ones((2, 2), np.float32)
    x = np.arange(3, dtype=np.int64)
    req = make_predict_elwcs_request("m", None, {"u": user}, {"x": x}, [2, 1], "elwcs", signature_name="rank", version_label="canary",
                                     output_filter=["score"])
    want = PredictRequest()
    want.model_spec.name = "m"
    want.model_spec.signature_name = "rank"
    want.model_spec.version_label = "canary"
    t = want.inputs["elwcs"]
    t.dtype = 7
    t.tensor_shape.dim.add().size = 2
    t.string_val.extend(e.SerializeToString(deterministic=True) for e in elwcs_from_input_dict({"u": user}, {"x": x}, [2, 1]))
    want.output_filter.append("score")
    assert req.SerializeToString(deterministic=True) == want.SerializeToString(deterministic=True)
    # each string: 42 vi(elwc) {0A vi(ex) ex}* 12 vi(ctx) ctx
    for s, e in zip(t.string_val, elwcs_from_input_dict({"u": user}, {"x": x}, [2, 1])):
        assert s[0] == 0x0A and s[-(e.context.ByteSize() + 2):][0] == 0x12


def test_one_query_equals_the_single_elwc_form():
    from min_tfs_client.codec import _host_example_request

    x = np.arange(8, dtype=np.float32).reshape(4, 2)
    ctx = {"u": np.arange(3, dtype=np.int64)}
    one = make_predict_elwcs_request("m", 4, {"u": ctx["u"][None]}, {"x": x}, [4], "in").SerializeToString(deterministic=True)
    assert one == _host_example_request("m", 4, {"x": x}, False, "in", ctx)


# ---- C ABI host arithmetic --------------------------------------------------------------------------------------------------
def _structs(input_dict, context_dict, sizes, kind=N.EXAMPLES_PREDICT_ELWCS, version=3, flags=0):
    sizes = np.asarray(sizes, np.int64)
    n, preps = _example_columns(input_dict)
    n = int(sizes.sum()) if sizes.size else n
    _, cpreps = _example_columns(context_dict) if context_dict else (0, [])
    feats = (N.Feature * max(len(preps), 1))(*[p[0] for p in preps])
    cfeats = (N.Feature * max(len(cpreps), 1))(*[p[0] for p in cpreps])
    req = N.ExampleRequest(model_name=b"m", model_name_len=1, has_version=1, order=N.ORDER_UPB, version=version, n_examples=n,
                           n_features=len(preps), flags=flags, features=feats)
    tg = N.ExampleTarget(kind=kind, key=b"q", key_len=1)
    ls = N.ExampleLists(list_sizes=sizes.ctypes.data if sizes.size else None, n_lists=sizes.size, context=cfeats,
                        n_context=len(cpreps), present=1)
    keep = (preps, cpreps, feats, cfeats, sizes)
    lbs = [p.bytes_entry or N.Bytes() for p in cpreps]
    lrg = [p[3] or N.Ragged() for p in cpreps]
    bs = [p.bytes_entry or N.Bytes() for p in preps]
    return req, tg, ls, keep, bs, lrg, lbs


def _arena(lib, req, tg, ls, bs=None, lrg=None, lbs=None, cx=None, tk=None, sq=None):
    cap = C.c_uint64()
    arr = lambda t, v: (t * max(len(v), 1))(*v) if v else None  # noqa: E731
    rc = lib.b200tfs_example_lists_arena_size(1, C.byref(req), None, arr(N.Bytes, bs), C.byref(tg), cx, None, tk, sq, None,
                                              C.byref(ls) if ls is not None else None, arr(N.Ragged, lrg), arr(N.Bytes, lbs), C.byref(cap))
    return rc, cap.value


@pytest.mark.parametrize("sizes", [[], [0], [3, 0, 2], [1] * 200, [130], [0] * 50 + [5]])
@pytest.mark.parametrize("ctx", ["none", "dense", "int"])
def test_request_size_and_arena_bound(sizes, ctx):
    lib = N.load()
    n = sum(sizes)
    x = np.linspace(-1, 1, 6 * n, dtype=np.float32).reshape(n, 6)
    cd = {} if ctx == "none" else {"u": np.ones((len(sizes), 40), np.float32)} if ctx == "dense" else \
        {"i": np.full((len(sizes), 5), -1, np.int64)}
    want = make_predict_elwcs_request("m", 3, cd, {"x": x}, sizes, "q").ByteSize()
    req, tg, ls, keep, bs, lrg, lbs = _structs({"x": x}, cd, sizes)
    size = C.c_uint64()
    rc = lib.b200tfs_example_lists_request_size(C.byref(req), C.byref(tg), None, None, None, None, None, C.byref(ls), None, C.byref(size))
    if ctx == "int":
        assert rc == N.E_ARG
    else:
        assert rc == N.OK and size.value == want
    rc, cap = _arena(lib, req, tg, ls, lrg=lrg, lbs=lbs)
    assert rc == N.OK and cap >= want


def test_arena_bound_covers_bytes_and_ragged_contexts():
    lib = N.load()
    rng = np.random.default_rng(1)
    sizes = [2, 0, 3]
    strs = [bytes(rng.integers(0, 256, k, dtype=np.uint8)) for k in (0, 300, 5)]
    text = BytesColumn.from_array(np.array(strs, object).astype("S300"))
    toks = RaggedColumn(np.full((3, 6), -(1 << 62), np.int64), np.array([6, 0, 3]))
    ids = RaggedColumn(np.full((5, 4), 1 << 60, np.int64), np.array([4, 4, 0, 1, 2]))
    cd, d = {"text": text, "toks": toks}, {"ids": ids}
    want = make_predict_elwcs_request("m", 3, cd, d, sizes, "q").ByteSize()
    req, tg, ls, keep, bs, lrg, lbs = _structs(d, cd, sizes)
    rc, cap = _arena(lib, req, tg, ls, bs=bs, lrg=lrg, lbs=lbs)
    assert rc == N.OK and cap >= want


def test_refusals():
    lib = N.load()
    x = {"x": np.zeros((3, 1), np.float32)}
    cd = {"u": np.zeros((2, 1), np.float32)}

    def arena(**over):
        req, tg, ls, keep, bs, lrg, lbs = _structs(x, cd, [2, 1])
        for k, v in over.items():
            obj = {"req": req, "tg": tg, "ls": ls}[k.split("_", 1)[0]]
            setattr(obj, k.split("_", 1)[1], v)
        return _arena(lib, req, tg, ls, lrg=lrg, lbs=lbs)[0]

    assert arena() == N.OK
    assert arena(ls_present=2) == N.E_ARG
    assert arena(ls_present=0) == N.E_ARG                       # PREDICT_ELWCS without its entry
    assert arena(tg_kind=N.EXAMPLES_PREDICT_STRING) == N.E_ARG  # the entry on another kind
    assert arena(ls_n_lists=-1) == N.E_ARG
    assert arena(ls_list_sizes=None) == N.E_ARG
    assert arena(ls_n_context=-1) == N.E_ARG
    assert arena(req_n_examples=4) == N.E_ARG                   # sum(list_sizes) != n_examples
    neg = np.array([4, -1], np.int64)
    assert arena(ls_list_sizes=neg.ctypes.data) == N.E_ARG
    huge = np.array([1 << 62, 1 << 62], np.int64)
    assert arena(ls_list_sizes=huge.ctypes.data) == N.E_ARG
    # beside a context, tasks or a sequence
    req, tg, ls, keep, bs, lrg, lbs = _structs(x, cd, [2, 1])
    cxf = (N.Feature * 1)(N.Feature(data=None, src_dtype=1, flags=0, row_elems=0, key=b"c", key_len=1))
    cx = N.ExampleContext(features=cxf, n_features=1, present=1)
    assert _arena(lib, req, tg, ls, cx=C.byref(cx))[0] == N.E_ARG
    task = (N.InferenceTask * 1)(N.InferenceTask(signature_name=None, signature_len=0, method=N.RESP_REGRESS))
    tk = N.ExampleTasks(tasks=C.addressof(task), n_tasks=1)
    assert _arena(lib, req, tg, ls, tk=C.byref(tk))[0] == N.E_ARG
    sq = N.ExampleSequence(present=1, n_context=0)
    assert _arena(lib, req, tg, ls, sq=C.byref(sq))[0] == N.E_ARG
    # the _specs_ entry points know no lists: PREDICT_ELWCS there is refused
    cap = C.c_uint64()
    assert lib.b200tfs_example_specs_arena_size(1, C.byref(req), None, None, C.byref(tg), None, None, None, None, None,
                                                C.byref(cap)) == N.E_ARG
    # malformed ragged and bytes context entries
    bad_rag = [N.Ragged(lengths=keep[4].ctypes.data, max_len=2, unit=1)]      # row_elems 1 != 2 * 1
    assert _arena(lib, req, tg, ls, lrg=bad_rag)[0] == N.E_ARG
    strs = {"s": BytesColumn.from_array(np.array([b"a", b"b"], "S1"))}
    req2, tg2, ls2, keep2, bs2, lrg2, lbs2 = _structs(x, strs, [2, 1])
    assert _arena(lib, req2, tg2, ls2)[0] == N.E_DTYPE                       # a DT_STRING context without its bytes entry
    lbs2[0].data_len = -1
    assert _arena(lib, req2, tg2, ls2, lbs=lbs2)[0] == N.E_ARG
    # a context feature with a leading dim that is not Q is refused by the Python layer; a request over 2 GiB is TOOBIG
    big = N.ExampleLists(list_sizes=None, n_lists=0, context=None, n_context=0, present=1)
    reqb, tgb, _, keepb, _, _, _ = _structs({"x": np.zeros((0, 1 << 28), np.float32)}, {}, [])
    reqb.n_examples = 40
    szs = np.full(40, 1, np.int64)
    big.list_sizes, big.n_lists = szs.ctypes.data, 40
    assert _arena(lib, reqb, tgb, big)[0] == N.E_TOOBIG
