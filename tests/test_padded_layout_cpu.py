"""b200tfs_padded_layout: the padded dtype / shape / bytes of a batch with ragged trailing dims, computed on the host without a
device, against the numpy definition (rows summed, every trailing axis the batch maximum)."""
import ctypes as C

import numpy as np
import pytest

from min_tfs_client import _native as N
from oracle import wire_oracle as O


def layout(wires, keys, cast=0):
    lib = N.load()
    offs, cur = [], 0
    for w in wires:
        offs.append(cur)
        cur += len(w)
    n, nk = len(wires), len(keys)
    pk = (N.PadKey * nk)()
    kb = [k.encode() for k in keys]
    for i, k in enumerate(kb):
        pk[i].key, pk[i].key_len = k, len(k)
    N.check(lib.b200tfs_padded_layout(C.c_char_p(b"".join(wires)), n, (C.c_uint64 * n)(*offs), (C.c_uint64 * n)(*[len(w) for w in wires]),
                                      nk, pk, cast))
    return [(pk[i].status, pk[i].bad_rec, pk[i].dtype, tuple(pk[i].dims[d] for d in range(pk[i].rank)), pk[i].bytes) for i in range(nk)]


def padded_shape(parts):
    rank = parts[0].ndim
    return (sum(p.shape[0] for p in parts),) + tuple(max(p.shape[d] for p in parts) for d in range(1, rank))


DTYPES = [np.float32, np.float64, np.int32, np.int64, np.uint8, np.int8, np.int16, np.uint16, np.uint32, np.uint64, np.bool_,
          np.float16, np.complex64, np.complex128]


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: np.dtype(d).name)
def test_rows_and_per_axis_maxima(dtype):
    shapes = [(1, 4, 2), (0, 7, 1), (3, 2, 5), (1, 0, 3), (2, 6, 2)]
    parts = [np.ones(s, dtype) for s in shapes]
    wires = [O.build_predict_response([("z", np.zeros(1, np.float32)), ("y", p)]) for p in parts]
    st, bad, dt, shape, nb = layout(wires, ["y"])[0]
    want = padded_shape(parts)
    assert (st, bad, shape) == (N.OK, -1, want)
    assert nb == int(np.prod(want)) * np.dtype(dtype).itemsize
    assert dt == O._dt_of(parts[0])


def test_rank_one_is_the_concatenation_and_equal_shapes_agree_with_the_concat_layout():
    import test_concat_layout_cpu as CL

    for shapes in ([(3,), (0,), (5,)], [(2, 4), (1, 4), (3, 4)]):
        wires = [O.build_predict_response([("a", np.ones(s, np.float32))]) for s in shapes]
        assert layout(wires, ["a"]) == CL.layout(wires, ["a"])


@pytest.mark.parametrize("cast", [0, 19, 14])
def test_bytes_with_and_without_a_narrowing_cast(cast):
    parts = [np.ones((1, t, 8), np.float32) for t in (5, 17, 3)]
    ids = [np.ones((1, t), np.int64) for t in (5, 17, 3)]
    wires = [O.build_predict_response([("logits", p), ("ids", i)]) for p, i in zip(parts, ids)]
    (_, _, _, ls, lb), (_, _, _, is_, ib) = layout(wires, ["logits", "ids"], cast)
    assert ls == (3, 17, 8) and is_ == (3, 17)
    assert lb == 3 * 17 * 8 * (2 if cast else 4)
    assert ib == 3 * 17 * 8          # only float32 narrows


def test_every_problem_class():
    f = lambda *s: np.ones(s, np.float32)  # noqa: E731
    good = O.build_predict_response([("a", f(2, 3))])
    assert layout([good, O.build_predict_response([("a", f(2, 4))])], ["a"])[0][:2] == (N.OK, -1)   # other trailing dims: padded
    assert layout([good, O.build_predict_response([("b", f(2, 3))])], ["a"])[0][:2] == (N.E_KEY, 1)
    assert layout([good, O.build_predict_response([("a", f(2, 3, 1))])], ["a"])[0][:2] == (N.E_SHAPE, 1)
    assert layout([good, O.build_predict_response([("a", np.ones((2, 3), np.float64))])], ["a"])[0][:2] == (N.E_DTYPE, 1)
    assert layout([good, O.build_predict_response([("a", np.float32(1))])], ["a"])[0][:2] == (N.E_SHAPE, 1)
    st, bad = layout([good, good, good[:-3]], ["a"])[0][:2]      # a record that does not walk
    assert st != N.OK and bad == 2
    deep = O.build_predict_response([("a", np.ones((1,) * 20, np.float32))])
    assert layout([good, deep], ["a"])[0][:2] == (N.E_NONCANONICAL, 1)
    assert layout([O.build_predict_response([(f"k{i}", f(1)) for i in range(9)])], ["k0"])[0][:2] == (N.E_NONCANONICAL, 0)
    # the first problem in record order
    res = layout([good, O.build_predict_response([("a", np.ones((2, 3), np.int32))]), O.build_predict_response([("b", f(1))])], ["a"])
    assert res[0][:2] == (N.E_DTYPE, 1)
