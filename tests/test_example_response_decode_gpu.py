"""Classify / Regress responses decoded on the GPU (b200tfs_decode_example_responses, Codec.decode_*_responses): every case
compares against the definition built from ClassificationResponse.FromString / RegressionResponse.FromString, bit for bit."""
import ctypes as C
import struct

import numpy as np
import pytest

import cast_sweep as CS
import example_response_corpus as X
from devutil import Dev
from min_tfs_client import _native as N

pytestmark = pytest.mark.gpu


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _check(codec, kind, wires, **kw):
    calls = codec.example_response_device_calls
    vals, labels, counts = X.expected(kind, wires)
    if kind == X.REGRESS:
        got = codec.decode_regression_responses(wires, **kw)
        v = got.values
    else:
        got = codec.decode_classification_responses(wires, **kw)
        v = got.scores
        assert got.labels() == labels
        same = all(r == labels[0] for r in labels)
        assert got.class_labels == ((list(labels[0]) if labels else []) if same else None)
    host = v.copy_to_host() if hasattr(v, "copy_to_host") else np.asarray(v.cpu() if hasattr(v, "cpu") else v)
    assert host.shape == vals.shape and np.array_equal(_bits(host), _bits(vals))
    assert got.counts.tolist() == counts
    assert codec.example_response_device_calls == calls + 1, "the device route did not finish"
    return got


def test_regress_batches(codec):
    rng = np.random.default_rng(3)
    pats = CS.f32_patterns()
    for n in (1, 3, 257):
        wires = []
        for i in range(n):
            k = int(rng.integers(0, 40)) if i % 5 else 0
            bits = pats[rng.integers(0, len(pats), k)]
            wires.append(X.serialize(X.regression_nodes([struct.unpack("<f", struct.pack("<I", int(b)))[0] for b in bits])))
        _check(codec, X.REGRESS, wires)


def test_every_float_pattern_as_value_and_score(codec):
    pats = CS.f32_patterns()
    vals = [X.f32(int(b)) for b in pats]
    wire = X.serialize([(1, X.LEN, [(1, X.LEN, [] if v == b"\0\0\0\0" else [(1, X.I32, v)]) for v in vals])])
    got = _check(codec, X.REGRESS, [wire])
    assert np.array_equal(_bits(got.values), CS.quiet(pats.astype(np.uint32)))
    cls = X.serialize([(1, X.LEN, [(1, X.LEN, [(1, X.LEN, [(1, X.LEN, b"s")] + ([] if v == b"\0\0\0\0" else [(2, X.I32, v)]))])
                                   for v in vals])])
    got = _check(codec, X.CLASSIFY, [cls])
    assert got.class_labels == ["s"]


def test_one_response_of_65536_regressions(codec):
    rng = np.random.default_rng(4)
    _check(codec, X.REGRESS, [X.random_regression(rng, 65536)])


@pytest.mark.parametrize("ncls", [0, 1, 2, 1000])
def test_classify_class_counts(codec, ncls):
    rng = np.random.default_rng(ncls)
    labels = [f"class_{k}" for k in range(ncls)]
    wires = [X.random_classification(rng, n, labels) for n in (5, 0, 3)]
    got = _check(codec, X.CLASSIFY, wires)
    assert got.scores.shape == (8, ncls) and got.class_labels == labels


def test_classify_labels_that_differ(codec):
    rng = np.random.default_rng(8)
    wires = [X.random_classification(rng, 40, lambda i: [f"top{(i * 7 + k) % 13}" for k in range(5)]) for _ in range(257)]
    got = _check(codec, X.CLASSIFY, wires)
    assert got.class_labels is None
    wires = [X.random_classification(rng, 4, ["", "ß", "€uro", "😀", "plain"]) for _ in range(3)]
    assert _check(codec, X.CLASSIFY, wires).class_labels == ["", "ß", "€uro", "😀", "plain"]


def test_ragged_class_counts_raise(codec):
    rng = np.random.default_rng(9)
    wires = [X.random_classification(rng, 2, ["a", "b"]), X.random_classification(rng, 2, ["a"])]
    with pytest.raises(ValueError, match="number of classes"):
        codec.decode_classification_responses(wires)


def test_edge_cases_and_mutants_match_the_runtime(codec):
    """Every case of the CPU corpus through the kernels: the status the host walk gives, and what FromString raises."""
    from google.protobuf.message import DecodeError

    dev = Dev()
    lib = dev.lib
    try:
        cases = [(k, w) for _, k, w in X.edge_cases()] + X.mutants()
        cap = max(len(w) for _, w in cases)
        vdst = dev.malloc(4 * cap)
        ldst = dev.malloc(8 * cap)
        per, batch = (C.c_int64 * 3)(), (C.c_int64 * 5)()
        counts = {}
        for kind, wire in cases:
            try:
                X.expected(kind, [wire])
                want = N.OK
            except DecodeError:
                want = N.E_PARSE
            except ValueError:
                want = N.E_SHAPE
            w = np.frombuffer(wire + b"\0", np.uint8)
            off, ln = (C.c_uint64 * 1)(0), (C.c_uint64 * 1)(len(wire))
            N.check(lib.b200tfs_decode_example_responses_host_async(dev.ctx, kind, w.ctypes.data, 1, off, ln, vdst, cap, ldst, cap))
            N.check(lib.b200tfs_example_response_results(dev.ctx, 1, per, None, batch))
            assert per[2] == want and batch[3] == want, (wire.hex(), per[2], want)
            counts[want] = counts.get(want, 0) + 1
        assert counts[N.OK] > 100 and counts[N.E_PARSE] > 100
    finally:
        dev.close()
    for kind, wire in X.mutants()[::17]:
        fn = codec.decode_regression_responses if kind == X.REGRESS else codec.decode_classification_responses
        try:
            X.expected(kind, [wire])
        except (DecodeError, ValueError) as e:
            with pytest.raises(type(e)):
                fn([wire])
            continue
        fn([wire])


def test_stores_stay_inside_the_used_rows_and_the_capacities():
    dev = Dev()
    lib = dev.lib
    try:
        rng = np.random.default_rng(11)
        wires = [X.random_classification(rng, n, ["a", "bb", "c"]) for n in (4, 0, 6)]
        rows, ncls = 10, 3
        blob = b"".join(w.ljust((len(w) + 255) & ~255, b"\0") for w in wires)
        offs = np.cumsum([0] + [(len(w) + 255) & ~255 for w in wires[:-1]]).astype(np.uint64)
        off = (C.c_uint64 * 3)(*offs.tolist())
        ln = (C.c_uint64 * 3)(*[len(w) for w in wires])
        w = np.frombuffer(blob, np.uint8)
        per, batch = (C.c_int64 * 9)(), (C.c_int64 * 5)()
        canary = np.full(64, 0xA5A5A5A5, np.uint32)
        for vcap, lcap in ((64, 64), (17, 64), (64, 20), (0, 0)):
            v, lab = dev.upload(canary), dev.upload(np.tile(canary, 2))
            N.check(lib.b200tfs_decode_example_responses_host_async(dev.ctx, X.CLASSIFY, w.ctypes.data, 3, off, ln, v if vcap else None,
                                                                    vcap, lab if lcap else None, lcap))
            N.check(lib.b200tfs_example_response_results(dev.ctx, 3, per, None, batch))
            got_v, got_l = dev.download(v, 256, np.uint32), dev.download(lab, 512, np.uint32)
            used = rows * ncls
            assert (got_v[min(used, vcap):] == 0xA5A5A5A5).all() and (got_l[2 * min(used, lcap):] == 0xA5A5A5A5).all()
            fits = used <= vcap and used <= lcap
            assert batch[0] == rows and batch[1] == ncls and (batch[3] == N.OK) == fits
            if not fits:
                assert batch[3] == N.E_SIZE
        wires = [X.random_regression(rng, n) for n in (7, 9)]
        blob = b"".join(w.ljust((len(w) + 255) & ~255, b"\0") for w in wires)
        off = (C.c_uint64 * 2)(0, (len(wires[0]) + 255) & ~255)
        ln = (C.c_uint64 * 2)(*[len(x) for x in wires])
        w = np.frombuffer(blob, np.uint8)
        for vcap in (16, 7, 3):
            v = dev.upload(canary)
            N.check(lib.b200tfs_decode_example_responses_host_async(dev.ctx, X.REGRESS, w.ctypes.data, 2, off, ln, v, vcap, None, 0))
            N.check(lib.b200tfs_example_response_results(dev.ctx, 2, per, None, batch))
            got_v = dev.download(v, 256, np.uint32)
            assert (got_v[min(16, vcap):] == 0xA5A5A5A5).all()
            assert [per[2], per[5]] == [N.OK if vcap >= 7 else N.E_SIZE, N.OK if vcap >= 16 else N.E_SIZE]
    finally:
        dev.close()


def test_destinations_agree(codec):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(12)
    wires = [X.random_classification(rng, n, ["x", "y", "z"]) for n in (3, 5)]
    ref = codec.decode_classification_responses(wires).scores
    dev = codec.decode_classification_responses(wires, device=True).scores
    assert np.array_equal(_bits(dev.copy_to_host()), _bits(ref))
    t = torch.full((12, 3), 7.0, device="cuda")
    got = codec.decode_classification_responses(wires, out=t).scores
    torch.cuda.synchronize()
    assert tuple(got.shape) == (8, 3) and np.array_equal(_bits(got.cpu().numpy()), _bits(ref))
    assert (t[8:] == 7.0).all()
    pinned = codec.pinned_empty((10, 3))
    got = codec.decode_classification_responses(wires, out=pinned).scores
    assert got.shape == (8, 3) and np.shares_memory(got, pinned) and np.array_equal(_bits(got), _bits(ref))
    rw = [X.random_regression(rng, n) for n in (4, 6)]
    ref = codec.decode_regression_responses(rw).values
    t = torch.zeros(16, device="cuda")
    assert np.array_equal(_bits(codec.decode_regression_responses(rw, out=t).values.cpu().numpy()), _bits(ref))
    assert np.array_equal(_bits(codec.decode_regression_responses(rw, device=True).values.copy_to_host()), _bits(ref))
    small = torch.full((5,), 3.0, device="cuda")
    with pytest.raises(ValueError):
        codec.decode_regression_responses(rw, out=small)
    narrow = torch.full((12, 2), 3.0, device="cuda")
    with pytest.raises(ValueError):                      # C = 3
        codec.decode_classification_responses(wires, out=narrow)
    from google.protobuf.message import DecodeError

    with pytest.raises(DecodeError):
        codec.decode_regression_responses(rw + [rw[0][:-3]], out=torch.full((32,), 3.0, device="cuda"))
    torch.cuda.synchronize()
    assert (small == 3.0).all() and (narrow == 3.0).all(), "a call that raises wrote into out"
    exact = codec.device_array(np.zeros(10, np.float32))     # cannot be sliced: must have exactly the rows
    assert codec.decode_regression_responses(rw, out=exact).values is exact
    assert np.array_equal(_bits(exact.copy_to_host()), _bits(ref))
    with pytest.raises(ValueError):
        codec.decode_regression_responses(rw, out=codec.device_array(np.zeros(11, np.float32)))
    dev = codec.decode_regression_responses(rw, device=True).values
    assert dev.shape == (10,) and dev.nbytes == 40


def test_graph_replay_over_new_responses_of_the_same_lengths():
    """A captured decode replayed over new responses of the same record lengths: new row counts, values and labels."""
    dev = Dev()
    lib = dev.lib
    try:
        # 10 nonzero values (7 bytes each) and 35 zeros (2 bytes each) make results of the same length
        def reg(vals):
            return X.serialize(X.regression_nodes([float(v) for v in vals]))
        rng = np.random.default_rng(14)
        batches = [[reg(list(rng.standard_normal(10).astype(np.float32) + 5)), reg([0.0] * 35)],
                   [reg([0.0] * 35), reg(list(rng.standard_normal(10).astype(np.float32) + 5))],
                   [reg(list(rng.standard_normal(10).astype(np.float32) - 5)), reg(list(rng.standard_normal(10).astype(np.float32) + 9))]]
        lens = [len(w) for w in batches[0]]
        assert all([len(w) for w in b] == lens for b in batches)
        arena = dev.malloc(1024)
        off = (C.c_uint64 * 2)(0, 512)
        ln = (C.c_uint64 * 2)(*lens)
        vdst = dev.malloc(4 * 100)
        per, batch = (C.c_int64 * 6)(), (C.c_int64 * 5)()

        def load(b):
            img = np.zeros(1024, np.uint8)
            img[: lens[0]] = np.frombuffer(b[0], np.uint8)
            img[512: 512 + lens[1]] = np.frombuffer(b[1], np.uint8)
            N.check(lib.b200tfs_memcpy_h2d(dev.ctx, arena, img.ctypes.data, img.nbytes))

        load(batches[0])
        N.check(lib.b200tfs_decode_example_responses(dev.ctx, X.REGRESS, arena, 2, off, ln, vdst, 100, None, 0))
        N.check(lib.b200tfs_example_response_results(dev.ctx, 2, per, None, batch))
        N.check(lib.b200tfs_capture_begin(dev.ctx))
        N.check(lib.b200tfs_decode_example_responses(dev.ctx, X.REGRESS, arena, 2, off, ln, vdst, 100, None, 0))
        g = C.c_void_p()
        N.check(lib.b200tfs_capture_end(dev.ctx, C.byref(g)))
        for b in batches:
            load(b)
            N.check(lib.b200tfs_graph_launch(dev.ctx, g))
            N.check(lib.b200tfs_example_response_results(dev.ctx, 2, per, None, batch))
            vals, _, counts = X.expected(X.REGRESS, b)
            assert [per[1], per[4]] == counts and batch[0] == sum(counts) and batch[3] == N.OK
            assert np.array_equal(dev.download(vdst, 4 * batch[0], np.uint32), _bits(vals))
        N.check(lib.b200tfs_graph_destroy(g))
    finally:
        dev.close()


def _padded(wires, target):
    """Each response padded to `target` bytes with an unknown top-level field (skipped by the decode)."""
    out = []
    for w in wires:
        k = target - len(w) - 3
        assert 0 <= k < 1 << 14
        out.append(w + bytes([15 << 3 | 2]) + X.varint(k, 1 if k < 128 else 0) + b"\x00" * k)
        assert len(out[-1]) == target
    return out


def test_classify_graph_replay_over_new_labels_and_class_counts():
    """A captured Classify decode replayed over new responses of the same lengths: new rows, class counts, scores, labels and
    same_labels."""
    dev = Dev()
    lib = dev.lib
    try:
        rng = np.random.default_rng(16)
        batches = [[X.random_classification(rng, 3, ["a", "b"]), X.random_classification(rng, 2, ["a", "b"])],
                   [X.random_classification(rng, 1, ["x", "y", "z", "w"]), X.random_classification(rng, 4, lambda i: [f"{i}", "q", "r", "s"])],
                   [X.random_classification(rng, 0, []), X.random_classification(rng, 6, ["é", "ü", "ß"])]]
        batches = [_padded(b, 400) for b in batches]
        arena = dev.malloc(1024)
        off = (C.c_uint64 * 2)(0, 512)
        ln = (C.c_uint64 * 2)(400, 400)
        cap = 400
        vdst, ldst = dev.malloc(4 * cap), dev.malloc(8 * cap)
        per, batch = (C.c_int64 * 6)(), (C.c_int64 * 5)()

        def load(b):
            img = np.zeros(1024, np.uint8)
            img[:400] = np.frombuffer(b[0], np.uint8)
            img[512:912] = np.frombuffer(b[1], np.uint8)
            N.check(lib.b200tfs_memcpy_h2d(dev.ctx, arena, img.ctypes.data, img.nbytes))
            return img

        load(batches[0])
        N.check(lib.b200tfs_decode_example_responses(dev.ctx, X.CLASSIFY, arena, 2, off, ln, vdst, cap, ldst, cap))
        N.check(lib.b200tfs_example_response_results(dev.ctx, 2, per, None, batch))
        N.check(lib.b200tfs_capture_begin(dev.ctx))
        N.check(lib.b200tfs_decode_example_responses(dev.ctx, X.CLASSIFY, arena, 2, off, ln, vdst, cap, ldst, cap))
        g = C.c_void_p()
        N.check(lib.b200tfs_capture_end(dev.ctx, C.byref(g)))
        for b in batches:
            img = load(b)
            N.check(lib.b200tfs_graph_launch(dev.ctx, g))
            N.check(lib.b200tfs_example_response_results(dev.ctx, 2, per, None, batch))
            scores, labels, counts = X.expected(X.CLASSIFY, b)
            rows, ncls = scores.shape
            assert [per[1], per[4]] == counts and list(batch)[:4] == [rows, ncls, int(all(r == labels[0] for r in labels)), N.OK]
            assert np.array_equal(dev.download(vdst, 4 * rows * ncls, np.uint32), _bits(scores).ravel())
            refs = dev.download(ldst, 8 * rows * ncls, np.uint32).reshape(-1, 2)
            base = [0] * counts[0] + [512] * counts[1]
            got = [[img[base[i] + refs[i * ncls + k, 0]: base[i] + refs[i * ncls + k, 0] + refs[i * ncls + k, 1]].tobytes().decode()
                    for k in range(ncls)] for i in range(rows)]
            assert got == labels
        N.check(lib.b200tfs_graph_destroy(g))
    finally:
        dev.close()


def test_grpc_round_trip():
    import grpc
    from fake_server import IdentityServer
    from min_tfs_client.codec import get_codec
    from min_tfs_client.requests import (CLASSIFY_METHOD, REGRESS_METHOD, gpu_classification_response_deserializer,
                                         gpu_example_request_serializer, gpu_regression_response_deserializer)
    from tensorflow_serving.apis.classification_pb2 import ClassificationResponse
    from tensorflow_serving.apis.regression_pb2 import RegressionResponse

    srv = IdentityServer()
    try:
        rng = np.random.default_rng(15)
        d = {"x": rng.standard_normal((20, 3)).astype(np.float32), "id": np.arange(20)}
        ch = grpc.insecure_channel(f"127.0.0.1:{srv.port}")
        calls = get_codec().example_response_device_calls
        cls = ch.unary_unary(CLASSIFY_METHOD, request_serializer=gpu_example_request_serializer,
                             response_deserializer=gpu_classification_response_deserializer)(("m", 4, d), timeout=30)
        reg = ch.unary_unary(REGRESS_METHOD, request_serializer=gpu_example_request_serializer,
                             response_deserializer=gpu_regression_response_deserializer)(("m", 4, d), timeout=30)
        ref_c = ClassificationResponse.FromString(cls.SerializeToString())
        ref_r = RegressionResponse.FromString(reg.SerializeToString())
        want = np.array([[c.score for c in cl.classes] for cl in ref_c.result.classifications], np.float32)
        assert np.array_equal(_bits(cls.scores), _bits(want)) and cls.scores.shape == (20, 2)
        assert cls.labels() == [["positive", "negative"]] * 20
        assert np.array_equal(_bits(reg.values), _bits(np.array([r.value for r in ref_r.result.regressions], np.float32)))
        assert cls.model_spec.version.value == 4 and reg.model_spec.name == "m"
        assert get_codec().example_response_device_calls == calls + 2
        ch.close()
    finally:
        srv.stop()
