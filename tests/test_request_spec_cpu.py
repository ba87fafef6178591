"""ModelSpec.signature_name, ModelSpec.version_label and PredictRequest.output_filter on the PredictRequest encode routes, on the
host: the framing code of the immediate planner (b200tfs_request_frame_spec), of the deferred encode's frame_requests_kernel
(b200tfs_request_frame_deferred_spec) and of the padded encode's framing kernels (b200tfs_padded_request_frame_columns_spec), each
run on the host from the same inline source.  The reference is the protobuf runtime: the route's bytes without the fields,
parsed, given the fields and serialised with deterministic=True."""
import ctypes as C

import numpy as np
import pytest

from min_tfs_client import _native as N
from min_tfs_client.codec import _Prepared, _RequestSpec
from tensorflow_serving.apis import predict_pb2

SIGS = [None, "", "serving_default", "sigé中", "s" * 127, "t" * 128, "u" * 16384]
LABELS = [None, "", "canary"]
VERSIONS = [None, 0, 300]
FILTERS = [None, [], [""], ["b"], ["out%d" % i for i in range(1000)], ["b", "a", "b"]]


def _varint(v):
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def _grpc(b):
    return b"\x00" + len(b).to_bytes(4, "big") + b


def reference(base, sig, label, filt, grpc):
    """protobuf's bytes of the request `base` (the route's bytes without the fields) with the fields set."""
    body = base[5:] if grpc else base
    m = predict_pb2.PredictRequest.FromString(body)
    assert m.SerializeToString(deterministic=True) == body
    if sig is not None:
        m.model_spec.signature_name = sig
    if label is not None:
        m.model_spec.version_label = label
    if filt is not None:
        m.output_filter.extend(filt)
    out = m.SerializeToString(deterministic=True)
    return _grpc(out) if grpc else out


def _spec(sig, label, filt):
    s = _RequestSpec.of([], sig, label, filt)
    return (s, C.byref(s.struct)) if s else (None, None)


def _request(model, version, preps, grpc, order=N.ORDER_UPB):
    arr = (N.Tensor * max(len(preps), 1))(*[p.struct for p in preps])
    name = model.encode()
    req = N.Request(model_name=name, model_name_len=len(name), has_version=int(version is not None), order=order,
                    version=version or 0, n_inputs=len(preps), flags=N.RF_GRPC_FRAME if grpc else 0, inputs=arr)
    return req, (arr, name)


def _inputs():
    rng = np.random.default_rng(7)
    return [("image", rng.standard_normal((3, 5)).astype(np.float32)), ("words", np.array(["a", "bcé"])),
            ("weights", rng.standard_normal(70).astype(np.float32))]


def immediate_wire(model, version, sig, label, filt, grpc):
    lib = N.load()
    ins = _inputs()
    preps = [_Prepared(a, k.encode(), None, False, False) for k, a in ins]
    req, keep = _request(model, version, preps, grpc)
    s, sp = _spec(sig, label, filt)
    total = C.c_uint64()
    N.check(lib.b200tfs_request_size_spec(C.byref(req), sp, C.byref(total)))
    n = len(preps)
    cap = total.value
    buf = (C.c_uint8 * cap)()
    flen = C.c_uint64()
    poff, plen, perm = (C.c_uint64 * n)(), (C.c_uint64 * n)(), (C.c_int32 * n)()
    N.check(lib.b200tfs_request_frame_spec(C.byref(req), sp, buf, cap, C.byref(flen), poff, plen, perm))
    frame = bytes(buf)[: flen.value]
    out, at = bytearray(), 0
    for j in range(n):
        p = preps[perm[j]]
        pay = p.array.tobytes()
        assert plen[j] == len(pay)
        take = poff[j] - len(out)
        out += frame[at: at + take]
        at += take
        out += pay
    out += frame[at:]
    assert len(out) == total.value
    arena = C.c_uint64()
    N.check(lib.b200tfs_request_arena_size_spec(1, C.byref(req), sp, C.byref(arena)))
    assert arena.value >= total.value
    return bytes(out)


def deferred_wire(model, version, sig, label, filt, grpc):
    lib = N.load()
    rng = np.random.default_rng(3)
    ins = [("ids", rng.integers(-2**40, 2**40, 200)), ("mask", rng.integers(0, 300, 7).astype(np.int32)),
           ("x", rng.standard_normal(40).astype(np.float32))]
    preps = [_Prepared(a, k.encode(), None, False, False) for k, a in ins]
    req, keep = _request(model, version, preps, grpc)
    s, sp = _spec(sig, label, filt)
    n = len(preps)
    pay = [b"".join(_varint(int(v) & (2**64 - 1)) for v in a.ravel()) if a.dtype.kind == "i" else a.tobytes() for _, a in ins]
    packed = (C.c_uint64 * n)(*[len(b) for b in pay])
    need = C.c_uint64()
    N.check(lib.b200tfs_request_arena_size_spec(1, C.byref(req), sp, C.byref(need)))
    buf = (C.c_uint8 * need.value)()
    off, ln = C.c_uint64(), C.c_uint64()
    poff, plen = (C.c_uint64 * n)(), (C.c_uint64 * n)()
    # the deferred encode's arena (b200tfs_request_arena_size_spec) holds the worst-case slot: the frame fits it exactly
    N.check(lib.b200tfs_request_frame_deferred_spec(C.byref(req), sp, packed, buf, need.value, C.byref(off), C.byref(ln), poff, plen))
    raw = bytearray(bytes(buf))
    for i, b in enumerate(pay):
        assert plen[i] == len(b)
        if ins[i][1].dtype.kind == "i" and ins[i][1].size <= 32:
            assert bytes(raw[poff[i]: poff[i] + len(b)]) == b     # a tiny varint input is written by the framing code itself
        else:
            raw[poff[i]: poff[i] + len(b)] = b
    return bytes(raw[off.value: off.value + ln.value])


def padded_wire(model, version, sig, label, filt, grpc):
    lib = N.load()
    rng = np.random.default_rng(5)
    P = rng.standard_normal((4, 6)).astype(np.float32)
    L = rng.integers(-5, 2**33, (4, 3))
    ins = [("p", P, [3, 5]), ("lab", L, [2, 2])]
    preps, pins, pay = [], [], []
    rows = []
    for k, a, shp in ins:
        p = _Prepared(a, k.encode(), None, False, False)
        row = (C.c_int64 * len(shp))(*shp)
        rows.append(row)
        preps.append(p)
        pins.append(N.PadInput(shapes=C.cast(row, C.c_void_p), cols=len(shp)))
        box = a[: shp[0], : shp[1]]
        pay.append(box.tobytes() if a.dtype == np.float32 else b"".join(_varint(int(v) & (2**64 - 1)) for v in box.ravel()))
    req, keep = _request(model, version, preps, grpc)
    s, sp = _spec(sig, label, filt)
    n = len(preps)
    packed = (C.c_uint64 * n)(*[len(b) for b in pay])
    arena = C.c_uint64()
    N.check(lib.b200tfs_padded_request_columns_arena_size_spec(1, C.byref(req), None, sp, C.byref(arena)))
    buf = np.zeros(arena.value, np.uint8)
    rec_len = C.c_uint64()
    poff, plen = (C.c_uint64 * n)(), (C.c_uint64 * n)()
    N.check(lib.b200tfs_padded_request_frame_columns_spec(C.byref(req), (N.PadInput * n)(*pins), None, sp, packed, buf.ctypes.data,
                                                           buf.size, C.byref(rec_len), poff, plen))
    assert rec_len.value + 256 + 128 <= arena.value
    raw = bytearray(buf[: rec_len.value].tobytes())
    for i, b in enumerate(pay):
        assert plen[i] == len(b)
        raw[poff[i]: poff[i] + len(b)] = b
    return bytes(raw)


ROUTES = {"immediate": immediate_wire, "deferred": deferred_wire, "padded": padded_wire}
GRID = [(s, lab, v, FILTERS[(i * 7 + j * 3 + k) % len(FILTERS)])
        for i, s in enumerate(SIGS) for j, lab in enumerate(LABELS) for k, v in enumerate(VERSIONS) if not (lab is not None and v is not None)]


@pytest.mark.parametrize("route", list(ROUTES))
@pytest.mark.parametrize("grpc", [False, True])
@pytest.mark.parametrize("sig,label,version,filt", GRID)
def test_route_matches_protobuf(route, grpc, sig, label, version, filt):
    f = ROUTES[route]
    base = f("model", version, None, None, None, grpc)
    got = f("model", version, sig, label, filt, grpc)
    assert got == reference(base, sig, label, filt, grpc)


@pytest.mark.parametrize("route", list(ROUTES))
@pytest.mark.parametrize("filt", FILTERS)
def test_every_filter(route, filt):
    f = ROUTES[route]
    base = f("m", None, None, None, None, False)
    assert f("m", None, "sig", "canary", filt, False) == reference(base, "sig", "canary", filt, False)


def test_wire_bytes_of_the_issue():
    """model_spec {name m, signature_name sig, version_label canary} and output_filter b, a behind the inputs map."""
    lib = N.load()
    p = _Prepared(np.array([1], np.int64), b"x", None, False, False)
    p.struct.packed_len = 1
    req, keep = _request("m", None, [p], False)
    s, sp = _spec("sig", "canary", ["b", "a"])
    buf = (C.c_uint8 * 256)()
    flen = C.c_uint64()
    one = (C.c_uint64 * 1)()
    N.check(lib.b200tfs_request_frame_spec(C.byref(req), sp, buf, 256, C.byref(flen), one, (C.c_uint64 * 1)(), (C.c_int32 * 1)()))
    frame = bytes(buf)[: flen.value]
    wire = frame[: one[0]] + b"\x01" + frame[one[0]:]
    m = predict_pb2.PredictRequest.FromString(wire)
    assert (m.model_spec.name, m.model_spec.signature_name, m.model_spec.version_label, list(m.output_filter)) == \
        ("m", "sig", "canary", ["b", "a"])
    assert wire.startswith(bytes.fromhex("0a100a016d1a03736967220663616e617279"))
    assert wire.endswith(bytes.fromhex("1a01621a0161"))


@pytest.mark.parametrize("route", ["size", "deferred", "padded"])
def test_version_with_label_is_refused(route):
    lib = N.load()
    p = _Prepared(np.zeros(3, np.float32), b"x", None, False, False)
    req, keep = _request("m", 1, [p], False)
    spec = N.RequestSpec(version_label=b"canary", version_label_len=6)
    out = C.c_uint64()
    if route == "size":
        rc = lib.b200tfs_request_size_spec(C.byref(req), C.byref(spec), C.byref(out))
    elif route == "deferred":
        buf = (C.c_uint8 * 4096)()
        rc = lib.b200tfs_request_frame_deferred_spec(C.byref(req), C.byref(spec), None, buf, 4096, C.byref(out), C.byref(C.c_uint64()),
                                                     None, None)
    else:
        rc = lib.b200tfs_padded_request_columns_arena_size_spec(1, C.byref(req), None, C.byref(spec), C.byref(out))
    assert rc == N.E_ARG


@pytest.mark.parametrize("bad", ["sig_len", "sig_null", "label_null", "filter_count", "filter_null", "filter_len", "filter_name"])
def test_malformed_spec_is_refused(bad):
    lib = N.load()
    p = _Prepared(np.zeros(3, np.float32), b"x", None, False, False)
    req, keep = _request("m", None, [p], False)
    names = (C.c_char_p * 2)(b"a", None)
    lens = (C.c_int64 * 2)(1, 1)
    spec = N.RequestSpec(version_label_len=-1)
    if bad == "sig_len":
        spec.signature_len = -1
    elif bad == "sig_null":
        spec.signature_len = 3
    elif bad == "label_null":
        spec.version_label_len = 2
    elif bad == "filter_count":
        spec.n_output_filter = -1
    elif bad == "filter_null":
        spec.n_output_filter = 1
    elif bad == "filter_len":
        lens[0] = -1
        spec.output_filter, spec.output_filter_len, spec.n_output_filter = names, lens, 1
    else:
        spec.output_filter, spec.output_filter_len, spec.n_output_filter = names, lens, 2
    out = C.c_uint64()
    assert lib.b200tfs_request_size_spec(C.byref(req), C.byref(spec), C.byref(out)) == N.E_ARG
    assert lib.b200tfs_request_arena_size_spec(1, C.byref(req), C.byref(spec), C.byref(out)) == N.E_ARG
    assert lib.b200tfs_padded_request_columns_arena_size_spec(1, C.byref(req), None, C.byref(spec), C.byref(out)) == N.E_ARG


def test_null_spec_is_the_plain_entry_point():
    lib = N.load()
    p = _Prepared(np.arange(5, dtype=np.float32), b"x", None, False, False)
    req, keep = _request("m", 2, [p], True)
    a, b = C.c_uint64(), C.c_uint64()
    N.check(lib.b200tfs_request_size(C.byref(req), C.byref(a)))
    N.check(lib.b200tfs_request_size_spec(C.byref(req), None, C.byref(b)))
    assert a.value == b.value
    assert immediate_wire("m", 2, None, None, None, True) == reference(immediate_wire("m", 2, None, None, None, True), None, None, None, True)


def test_python_spec_checks():
    with pytest.raises(ValueError, match="oneof"):
        _RequestSpec.of([None, 3], version_label="canary")
    with pytest.raises(ValueError, match="UTF-8"):
        _RequestSpec.of([None], signature_name=b"\xff\xfe")
    with pytest.raises(ValueError, match="UTF-8"):
        _RequestSpec.of([None], version_label=b"\xc3")
    with pytest.raises(ValueError, match="UTF-8"):
        _RequestSpec.of([None], output_filter=["ok", b"\x80"])
    with pytest.raises(TypeError):
        _RequestSpec.of([None], output_filter="scores")
    assert _RequestSpec.of([1, None]) is None
    s = _RequestSpec.of([None], signature_name="é", version_label=b"", output_filter=[b"a", "中"])
    assert (s.struct.signature_len, s.struct.version_label_len, s.struct.n_output_filter) == (2, 0, 2)
    assert s.struct.output_filter_len[1] == 3


# ---- the tf.Example family: closed-form sizes against protobuf, and the refusals -------------------------------------------
def _example_request(version=None):
    x = np.arange(12, dtype=np.float32).reshape(4, 3)
    f = N.Feature(data=x.ctypes.data, src_dtype=1, flags=0, row_elems=3, key=b"x", key_len=1)
    feats = (N.Feature * 1)(f)
    req = N.ExampleRequest(model_name=b"m", model_name_len=1, has_version=int(version is not None), order=N.ORDER_UPB,
                           version=version or 0, n_examples=4, n_features=1, flags=0, features=feats)
    return req, (x, feats), {"x": x}


@pytest.mark.parametrize("sig,label,filt", [(None, None, None), ("classification", None, None), (None, "", None), ("s" * 200, "canary", None),
                                            ("p", "v", ["a", "", "a"]), (None, None, ["o%d" % i for i in range(300)])])
@pytest.mark.parametrize("kind", ["list", "predict", "tasks"])
def test_example_sizes(kind, sig, label, filt):
    from min_tfs_client.codec import _host_example_request
    from min_tfs_client.requests import CLASSIFY_METHOD_NAME, REGRESS_METHOD_NAME

    lib = N.load()
    req, keep, d = _example_request()
    target = N.ExampleTarget(kind=N.EXAMPLES_PREDICT_STRING, key=b"ex", key_len=2) if kind == "predict" else None
    task_arr = (N.InferenceTask * 2)(N.InferenceTask(signature_name=b"a", signature_len=1, method=N.RESP_CLASSIFY),
                                     N.InferenceTask(signature_name=b"", signature_len=0, method=N.RESP_REGRESS))
    tk = N.ExampleTasks(tasks=C.addressof(task_arr), n_tasks=2) if kind == "tasks" else None
    if kind == "tasks":
        sig = None
    s, sp = _spec(sig, label, filt)
    total = C.c_uint64()
    rc = lib.b200tfs_example_specs_request_size(C.byref(req), C.byref(target) if target else None, None, C.byref(tk) if tk else None,
                                                None, None, sp, C.byref(total))
    if filt is not None and kind != "predict":
        assert rc == N.E_ARG                 # output_filter is a PredictRequest field
        return
    N.check(rc)
    fields = {k: v for k, v in dict(signature_name=sig, version_label=label, output_filter=filt).items() if v is not None}
    tasks = [("a", CLASSIFY_METHOD_NAME), ("", REGRESS_METHOD_NAME)] if kind == "tasks" else None
    ref = _host_example_request("m", None, d, False, "ex" if kind == "predict" else None, None, tasks, **fields)
    assert total.value == len(ref)
    arena = C.c_uint64()
    N.check(lib.b200tfs_example_specs_arena_size(1, C.byref(req), None, None, C.byref(target) if target else None, None, None,
                                                 C.byref(tk) if tk else None, None, sp, C.byref(arena)))
    assert arena.value >= total.value


def test_example_refusals():
    lib = N.load()
    req, keep, _ = _example_request(version=2)
    total = C.c_uint64()
    label = N.RequestSpec(version_label=b"x", version_label_len=1)
    assert lib.b200tfs_example_specs_request_size(C.byref(req), None, None, None, None, None, C.byref(label), C.byref(total)) == N.E_ARG
    req, keep, _ = _example_request()
    task_arr = (N.InferenceTask * 1)(N.InferenceTask(signature_name=b"a", signature_len=1, method=N.RESP_CLASSIFY))
    tk = N.ExampleTasks(tasks=C.addressof(task_arr), n_tasks=1)
    sig = N.RequestSpec(signature_name=b"s", signature_len=1, version_label_len=-1)
    assert lib.b200tfs_example_specs_request_size(C.byref(req), None, None, C.byref(tk), None, None, C.byref(sig), C.byref(total)) == N.E_ARG
    names, lens = (C.c_char_p * 1)(b"y"), (C.c_int64 * 1)(1)
    filt = N.RequestSpec(version_label_len=-1, output_filter=names, output_filter_len=lens, n_output_filter=1)
    for t in (None, C.byref(tk)):
        assert lib.b200tfs_example_specs_request_size(C.byref(req), None, None, t, None, None, C.byref(filt), C.byref(total)) == N.E_ARG
    assert lib.b200tfs_example_specs_arena_size(1, C.byref(req), None, None, None, None, None, None, None, C.byref(filt),
                                                C.byref(total)) == N.E_ARG


def test_host_reference_helpers():
    from min_tfs_client.requests import CLASSIFY_METHOD_NAME, make_multi_inference_request, make_predict_sequence_examples_request

    d = {"x": np.ones((2, 1), np.float32)}
    m = make_multi_inference_request("m", None, [("a", CLASSIFY_METHOD_NAME)], d, version_label="canary")
    assert m.tasks[0].model_spec.version_label == "canary" and m.tasks[0].model_spec.signature_name == "a"
    for bad in (dict(signature_name="s"), dict(output_filter=["o"])):
        with pytest.raises(ValueError):
            make_multi_inference_request("m", None, [("a", CLASSIFY_METHOD_NAME)], d, **bad)
    p = make_predict_sequence_examples_request("m", None, {}, {"f": np.ones((2, 3), np.float32)}, "s", signature_name="sig",
                                               output_filter=["b", "a"])
    assert p.model_spec.signature_name == "sig" and list(p.output_filter) == ["b", "a"]
