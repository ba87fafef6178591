"""Host planner of the tf.Example requests (Classify / Regress), without a GPU: b200tfs_example_request_size against the
protobuf message's ByteSize(), b200tfs_example_arena_size against the serialised length, and refusals from dims alone."""
import ctypes as C

import numpy as np
import pytest

from min_tfs_client import _native as N
from min_tfs_client.codec import _example_columns
from min_tfs_client.requests import TensorServingClient
from tensorflow_serving.apis.classification_pb2 import ClassificationRequest

KEYS = ["a", "ab", "abc", "b", "", "été", "中", "x" * 200]


def _message(name, version, d):
    return TensorServingClient._make_example_request(None, ClassificationRequest, name, d, version)


def _struct(name, version, d, grpc_frame=False):
    n, preps = _example_columns(d)
    feats = (N.Feature * max(len(preps), 1))(*[p[0] for p in preps])
    nb = name.encode()
    req = N.ExampleRequest(model_name=nb, model_name_len=len(nb), has_version=int(version is not None), order=N.ORDER_UPB,
                           version=version or 0, n_examples=n, n_features=len(preps), flags=N.RF_GRPC_FRAME if grpc_frame else 0,
                           features=feats)
    return req, (preps, feats, nb)


def _random_dict(rng, n, kinds):
    d = {}
    for k in rng.choice(KEYS, size=rng.integers(0 if n == 0 else 1, 7), replace=False):
        width = int(rng.choice([0, 1, 7, 300]))
        kind = rng.choice(kinds)
        shape = () if rng.random() < 0.15 else (n,) if width == 1 and rng.random() < 0.5 else (n, width)
        if kind == "f":
            dt = rng.choice([np.float16, np.float32, np.float64])
            d[str(k)] = rng.standard_normal(shape).astype(dt)
        elif kind == "neg":
            d[str(k)] = -rng.integers(1, 1 << 62, size=shape, dtype=np.int64)
        else:
            dt = rng.choice([np.int8, np.int32, np.uint64, np.bool_])
            d[str(k)] = rng.integers(0, 2, size=shape).astype(dt) if dt is np.bool_ else \
                rng.integers(0, np.iinfo(dt).max, size=shape, dtype=dt)
    return d


@pytest.mark.parametrize("seed", range(40))
def test_size_equals_byte_size_float_only(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.choice([0, 1, 1000]))
    d = _random_dict(rng, n, ["f"])
    name = str(rng.choice(["", "m", "model-é"]))
    version = [None, 0, 7][seed % 3]
    lib = N.load()
    for grpc_frame in (False, True):
        req, keep = _struct(name, version, d, grpc_frame)
        total = C.c_uint64()
        N.check(lib.b200tfs_example_request_size(C.byref(req), C.byref(total)))
        assert total.value == _message(name, version, d).ByteSize() + (5 if grpc_frame else 0)
        arena = C.c_uint64()
        N.check(lib.b200tfs_example_arena_size(1, C.byref(req), C.byref(arena)))
        assert arena.value >= total.value


def test_size_of_empty_and_prefix_keys():
    lib = N.load()
    x = np.arange(6, dtype=np.float32).reshape(3, 2)
    for d in ({}, {"a": x, "ab": x, "abc": x[:, :0]}, {"s": np.float32(2.5)}, {"s": np.float64(2.5), "t": np.zeros(0, np.float16)}):
        req, keep = _struct("m", 3, d)
        total = C.c_uint64()
        N.check(lib.b200tfs_example_request_size(C.byref(req), C.byref(total)))
        assert total.value == _message("m", 3, d).ByteSize()


@pytest.mark.parametrize("seed", range(20))
def test_arena_bounds_requests_with_integer_columns(seed):
    rng = np.random.default_rng(100 + seed)
    n = int(rng.choice([1, 17, 500]))
    d = _random_dict(rng, n, ["f", "i", "neg"])
    d["neg_row"] = np.full((n, 9), -1, dtype=np.int64)       # ten bytes per element: the worst case itself
    lib = N.load()
    req, keep = _struct("m", 1, d, grpc_frame=True)
    total = C.c_uint64()
    assert lib.b200tfs_example_request_size(C.byref(req), C.byref(total)) == N.E_ARG
    assert b"integer" in lib.b200tfs_last_error()
    arena = C.c_uint64()
    N.check(lib.b200tfs_example_arena_size(1, C.byref(req), C.byref(arena)))
    assert arena.value >= len(_message("m", 1, d).SerializeToString(deterministic=True)) + 5


def test_too_big_is_refused_from_dims_alone():
    lib = N.load()
    key = b"dense"
    f = N.Feature(data=None, src_dtype=1, flags=0, row_elems=1 << 20, key=key, key_len=len(key))    # 4 MiB per example
    req = N.ExampleRequest(model_name=b"m", model_name_len=1, has_version=0, order=N.ORDER_UPB, version=0, n_examples=600,
                           n_features=1, flags=0, features=C.pointer(f))
    total, arena = C.c_uint64(), C.c_uint64()
    assert lib.b200tfs_example_request_size(C.byref(req), C.byref(total)) == N.E_TOOBIG
    assert lib.b200tfs_example_arena_size(1, C.byref(req), C.byref(arena)) == N.E_TOOBIG
    req.n_examples = 500                                     # 2 000 000 000 bytes and some framing: under the limit
    N.check(lib.b200tfs_example_request_size(C.byref(req), C.byref(total)))
    assert 2_000_000_000 < total.value < 2 ** 31 - 1
    f.src_dtype = 9                                          # int64: at least a byte per element, 10 at most
    req.n_examples = 2100
    assert lib.b200tfs_example_arena_size(1, C.byref(req), C.byref(arena)) == N.E_TOOBIG
    req.n_examples = 100
    N.check(lib.b200tfs_example_arena_size(1, C.byref(req), C.byref(arena)))
    assert arena.value >= 100 * 10 * (1 << 20)


def test_bad_arguments():
    lib = N.load()
    total = C.c_uint64()
    for dtype in (7, 8, 14, 18):                             # string, complex64, bfloat16, complex128
        f = N.Feature(data=None, src_dtype=dtype, flags=0, row_elems=1, key=b"k", key_len=1)
        req = N.ExampleRequest(model_name=b"", model_name_len=0, has_version=0, order=N.ORDER_UPB, version=0, n_examples=1,
                               n_features=1, flags=0, features=C.pointer(f))
        assert lib.b200tfs_example_request_size(C.byref(req), C.byref(total)) == N.E_DTYPE
    f = N.Feature(data=None, src_dtype=1, flags=0, row_elems=-1, key=b"k", key_len=1)
    req.features = C.pointer(f)
    assert lib.b200tfs_example_request_size(C.byref(req), C.byref(total)) == N.E_SHAPE
    f.row_elems = 1
    req.flags = 0x40
    assert lib.b200tfs_example_request_size(C.byref(req), C.byref(total)) == N.E_ARG
    req.flags, req.n_features = 0, 0                         # examples without features
    assert lib.b200tfs_example_request_size(C.byref(req), C.byref(total)) == N.E_ARG


def test_host_preparation_raises_like_examples_from_input_dict():
    from min_tfs_client.requests import examples_from_input_dict

    bad = {"a": np.zeros((2, 3), np.float32), "b": np.zeros((3,), np.int64)}
    with pytest.raises(ValueError, match="disagree") as ours:
        _example_columns(bad)
    with pytest.raises(ValueError) as ref:
        examples_from_input_dict(bad)
    assert str(ours.value) == str(ref.value)
    assert _example_columns({"s": np.array(["x", "y"])}) is None          # strings: the host assembles the request
    assert _example_columns({"c": np.zeros(2, np.complex64)}) is None     # ... and raises there
