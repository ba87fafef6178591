"""b200tfs_concat_layout: the concatenated dtype / shape / bytes of a batch, computed on the host without a device."""
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
    ck = (N.ConcatKey * nk)()
    kb = [k.encode() for k in keys]
    for i, k in enumerate(kb):
        ck[i].key, ck[i].key_len = k, len(k)
    N.check(lib.b200tfs_concat_layout(C.c_char_p(b"".join(wires)), n, (C.c_uint64 * n)(*offs), (C.c_uint64 * n)(*[len(w) for w in wires]),
                                      nk, ck, cast))
    return [(ck[i].status, ck[i].bad_rec, ck[i].dtype, tuple(ck[i].dims[d] for d in range(ck[i].rank)), ck[i].bytes) for i in range(nk)]


DTYPES = [np.float32, np.float64, np.int32, np.int64, np.uint8, np.int8, np.int16, np.uint16, np.uint32, np.uint64, np.bool_,
          np.float16, np.complex64, np.complex128]


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: np.dtype(d).name)
def test_layout_agrees_with_numpy(dtype):
    rows = [2, 0, 5, 1]
    parts = [np.ones((r, 3, 2), dtype) for r in rows]
    wires = [O.build_predict_response([("z", np.zeros(1, np.float32)), ("y", p)]) for p in parts]
    cat = np.concatenate(parts)
    st, bad, dt, shape, nb = layout(wires, ["y"])[0]
    assert (st, bad, shape, nb) == (N.OK, -1, cat.shape, cat.nbytes)
    assert dt == O._dt_of(parts[0])


def test_several_keys_map_orders_duplicates_and_the_cast():
    a = np.ones((2, 4), np.float32)
    b = np.ones((3,), np.int64)
    w1 = O.build_predict_response([("a", a), ("b", b)])
    w2 = O.build_predict_response([("b", b[:1]), ("a", np.ones((9, 4), np.float32))])
    w3 = O.build_predict_response([("a", np.ones((7, 4), np.float32)), ("a", a)])      # duplicate key: the last entry wins
    res = layout([w1, w2], ["b", "a"])
    assert res[0][3] == (4,) and res[1][3] == (11, 4) and res[1][4] == 11 * 16
    res = layout([w1, w3], ["a"], cast=19)
    assert res[0][:2] == (N.OK, -1) and res[0][3] == (4, 4) and res[0][4] == 4 * 4 * 2


def test_every_mismatch_class():
    f = lambda *s: np.ones(s, np.float32)  # noqa: E731
    good = O.build_predict_response([("a", f(2, 3))])
    assert layout([good, O.build_predict_response([("b", f(2, 3))])], ["a"])[0][:2] == (N.E_KEY, 1)
    assert layout([good, O.build_predict_response([("a", f(2, 4))])], ["a"])[0][:2] == (N.E_SHAPE, 1)
    assert layout([good, O.build_predict_response([("a", f(2, 3, 1))])], ["a"])[0][:2] == (N.E_SHAPE, 1)
    assert layout([good, O.build_predict_response([("a", np.ones((2, 3), np.float64))])], ["a"])[0][:2] == (N.E_DTYPE, 1)
    assert layout([good, O.build_predict_response([("a", np.float32(1))])], ["a"])[0][:2] == (N.E_SHAPE, 1)
    assert layout([good, good[:-3]], ["a"])[0][0] != N.OK
    deep = O.build_predict_response([("a", np.ones((1,) * 20, np.float32))])
    assert layout([deep], ["a"])[0][:2] == (N.E_NONCANONICAL, 0)
    assert layout([O.build_predict_response([(f"k{i}", f(1)) for i in range(9)])], ["k0"])[0][:2] == (N.E_NONCANONICAL, 0)
