"""b200tfs_padded_request_frame - the framing the padded encode's kernels write for one request, run on the host from the same
inline source - against b200tfs_request_frame of the request sliced out of the padded tensors on the host, and the arena bound
b200tfs_padded_request_arena_size against the exact records at the worst-case shapes."""
import ctypes as C

import numpy as np
import pytest

from min_tfs_client import _native as N
from min_tfs_client.codec import _Prepared

_DTYPES = [np.float32, np.float64, np.float16, np.complex64, np.complex128, np.bool_, np.int8, np.int16, np.int32, np.int64,
           np.uint8, np.uint16, np.uint32, np.uint64]
_VARINT = {np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint16, np.uint32, np.uint64, np.float16}


def _packed_len(a) -> int:
    a = np.ascontiguousarray(a)
    if a.dtype == np.float16:
        v = a.view(np.uint16).astype(np.uint64)
    else:
        v = a.astype(np.int64).view(np.uint64) if a.dtype.kind == "i" else a.astype(np.uint64)
    n = np.ones(v.shape, dtype=np.int64)
    for s in range(7, 64, 7):
        n += (v >> np.uint64(s)) != 0
    return int(n.sum())


def _request(name, version, preps, order, grpc):
    arr = (N.Tensor * max(len(preps), 1))(*[p.struct for p in preps])
    nb = name.encode()
    return N.Request(model_name=nb, model_name_len=len(nb), has_version=int(version is not None), order=order,
                     version=version or 0, n_inputs=len(preps), flags=N.RF_GRPC_FRAME if grpc else 0, inputs=arr), arr


def _check(padded, rows_of, broadcast, order=N.ORDER_UPB, grpc=False, version=7, content=False, packed_scale=None):
    """padded: {key: array}; rows_of: {key: the request's shape row (len m or 1)}; broadcast: {key: array}"""
    lib = N.load()
    sliced = {}
    for k, p in padded.items():
        s = rows_of[k]
        dims = list(s) + list(p.shape[len(s):])
        sliced[k] = p[tuple(slice(0, int(d)) for d in dims)]
    sliced.update(broadcast)
    keys = list(padded) + list(broadcast)
    # the sliced request, measured
    sp = [_Prepared(sliced[k], k.encode(), None, content, False) for k in keys]
    packed = [0] * len(keys)
    for i, k in enumerate(keys):
        if not content and sliced[k].dtype.type in _VARINT and sliced[k].size:
            packed[i] = _packed_len(sliced[k]) if packed_scale is None else packed_scale * sliced[k].size
            sp[i].struct.packed_len = packed[i]
    req, keep1 = _request("model", version, sp, order, grpc)
    cap = 1 << 16
    fbuf = np.zeros(cap, np.uint8)
    flen = C.c_uint64()
    n = len(keys)
    poff, plen, perm = (C.c_uint64 * max(n, 1))(), (C.c_uint64 * max(n, 1))(), (C.c_int32 * max(n, 1))()
    N.check(lib.b200tfs_request_frame(C.byref(req), fbuf.ctypes.data, cap, C.byref(flen), poff, plen, perm))
    # the padded request
    pp = [_Prepared(padded[k] if k in padded else broadcast[k], k.encode(), None, content, False) for k in keys]
    rows = []
    pins = []
    for i, k in enumerate(keys):
        if k in padded:
            r = (C.c_int64 * len(rows_of[k]))(*[int(x) for x in rows_of[k]])
            rows.append(r)
            pins.append(N.PadInput(shapes=C.cast(r, C.c_void_p), cols=len(rows_of[k])))
        else:
            pp[i].struct.flags |= N.F_BROADCAST
            pins.append(N.PadInput(shapes=None, cols=0))
    preq, keep2 = _request("model", version, pp, order, grpc)
    pin_arr = (N.PadInput * max(n, 1))(*pins)
    pk = (C.c_uint64 * max(n, 1))(*packed)
    total = int(flen.value) + sum(plen[i] for i in range(n))
    buf = np.full(total + 64, 0xEE, np.uint8)
    rec_len = C.c_uint64()
    qoff, qlen = (C.c_uint64 * max(n, 1))(), (C.c_uint64 * max(n, 1))()
    N.check(lib.b200tfs_padded_request_frame(C.byref(preq), pin_arr, pk, buf.ctypes.data, buf.size, C.byref(rec_len), qoff, qlen))
    assert rec_len.value == total
    # b200tfs_request_frame reports in wire order (perm), b200tfs_padded_request_frame per input
    assert [qoff[perm[j]] for j in range(n)] == [poff[j] for j in range(n)]
    assert [qlen[perm[j]] for j in range(n)] == [plen[j] for j in range(n)]
    # framing bytes = everything outside the payload ranges, in wire order; nothing written past the record
    mask = np.ones(total, bool)
    for i in range(n):
        mask[qoff[i]: qoff[i] + qlen[i]] = False
        assert (buf[qoff[i]: qoff[i] + qlen[i]] == 0xEE).all()
    assert buf[:total][mask].tobytes() == fbuf[: flen.value].tobytes()
    assert (buf[total:] == 0xEE).all()


@pytest.mark.parametrize("dtype", _DTYPES, ids=lambda d: np.dtype(d).name)
@pytest.mark.parametrize("rank", [1, 2, 3, 4, 16])
def test_frame_matches_sliced_request(dtype, rank):
    rng = np.random.default_rng(rank * 100 + _DTYPES.index(dtype))
    for trial in range(4):
        dims = [int(x) for x in rng.integers(0, 4 if rank == 16 else 9, size=rank)]
        dims[0] = int(rng.integers(0, 20))
        p = (rng.standard_normal(dims) * 1000).astype(dtype) if np.dtype(dtype).kind != "b" else rng.integers(0, 3, dims).astype(np.uint8).view(np.bool_)
        full = trial % 2 == 0
        row = [int(rng.integers(0, dims[0] + 1))] if not full else [int(rng.integers(0, dims[0] + 1))] + [int(rng.integers(0, d + 1)) for d in dims[1:]]
        _check({"x": p}, {"x": row}, {}, order=[N.ORDER_UPB, N.ORDER_GIVEN][trial % 2], grpc=trial == 3, content=trial == 2)


@pytest.mark.parametrize("axis", range(4))
def test_zero_dims_on_every_axis(axis):
    p = np.arange(5 * 4 * 3 * 2, dtype=np.float32).reshape(5, 4, 3, 2)
    row = [2, 3, 2, 1]
    row[axis] = 0
    _check({"x": p}, {"x": row}, {})
    _check({"ids": p.astype(np.int64)}, {"ids": row}, {})


@pytest.mark.parametrize("per", range(1, 11))
def test_varint_packed_lengths(per):
    p = np.arange(40, dtype=np.int64).reshape(8, 5)
    _check({"ids": p, "mask": p.astype(np.int32)}, {"ids": [3, 4], "mask": [3]}, {}, packed_scale=per)


@pytest.mark.parametrize("order", [N.ORDER_UPB, N.ORDER_GIVEN, N.ORDER_BYTES])
def test_keys_and_broadcast(order):
    rng = np.random.default_rng(order)
    padded = {"input_ids": rng.integers(-5, 50000, (16, 12)), "attention_mask": rng.integers(0, 2, (16, 12)).astype(np.int64),
              "emb": rng.standard_normal((16, 12, 4)).astype(np.float32)}
    rows = {"input_ids": [1, 7], "attention_mask": [1, 7], "emb": [1, 7, 4]}
    bc = {"temperature": np.float32(0.5).reshape(()), "input": np.array([3, -1], np.int32), "t": np.zeros((2, 0, 3), np.float64)}
    _check(padded, rows, bc, order=order)
    _check(padded, rows, bc, order=order, grpc=True, version=None)
    _check(padded, {"input_ids": [0], "attention_mask": [0, 3], "emb": [0, 2, 1]}, bc, order=order)


def test_arena_size_bounds_worst_case_records():
    lib = N.load()
    n, R = 8, 64
    P = {"ids": np.full((R, 32), -1, np.int64), "x": np.zeros((R, 16, 3), np.float32), "b": np.zeros((R,), np.bool_)}
    bc = {"s": np.full((5,), -1, np.int32)}
    keys = list(P) + list(bc)
    pp = [_Prepared(P[k] if k in P else bc[k], k.encode(), None, False, False) for k in keys]
    pp[-1].struct.flags |= N.F_BROADCAST
    req, keep = _request("m" * 300, 2 ** 62, pp, N.ORDER_UPB, True)
    cap = C.c_uint64()
    N.check(lib.b200tfs_padded_request_arena_size(n, C.byref(req), C.byref(cap)))
    # worst case: one request takes all rows at full trailing dims, every varint 10 bytes; the others are empty
    need = 0
    for r in range(n):
        rows = {"ids": [R if r == 0 else 0, 32], "x": [R if r == 0 else 0, 16, 3], "b": [R if r == 0 else 0]}
        pins, holds = [], []
        for k in keys:
            if k in P:
                h = (C.c_int64 * len(rows[k]))(*rows[k])
                holds.append(h)
                pins.append(N.PadInput(shapes=C.cast(h, C.c_void_p), cols=len(rows[k])))
            else:
                pins.append(N.PadInput(shapes=None, cols=0))
        pk = (C.c_uint64 * len(keys))(10 * R * 32 if r == 0 else 0, 0, 0, 50)
        rec_len = C.c_uint64()
        buf = np.zeros(1 << 20, np.uint8)
        N.check(lib.b200tfs_padded_request_frame(C.byref(req), (N.PadInput * len(keys))(*pins), pk, buf.ctypes.data, buf.size,
                                                 C.byref(rec_len), None, None))
        need = ((need + 255) & ~255) + 127 + rec_len.value
    assert cap.value >= need


def test_argument_errors():
    lib = N.load()
    p = np.zeros((4, 3), np.float32)
    pp = [_Prepared(p, b"x", None, False, False)]
    req, keep = _request("m", None, pp, N.ORDER_UPB, False)
    buf = np.zeros(4096, np.uint8)
    rl = C.c_uint64()

    def frame(row, cols=None):
        h = (C.c_int64 * len(row))(*row)
        pin = (N.PadInput * 1)(N.PadInput(shapes=C.cast(h, C.c_void_p), cols=len(row) if cols is None else cols))
        return lib.b200tfs_padded_request_frame(C.byref(req), pin, None, buf.ctypes.data, buf.size, C.byref(rl), None, None)

    assert frame([2, 3]) == N.OK
    assert frame([-1, 3]) == N.E_SHAPE
    assert frame([2, 4]) == N.E_SHAPE
    assert frame([5, 3]) == N.E_SIZE
    assert frame([2, 3, 1], cols=3) == N.E_ARG
    # DT_STRING, PRESERIALIZED, > 8 padded inputs, rank 0 padded, rank 17
    s = _Prepared(np.array(["a"]), b"s", None, False, False)
    for preps in ([s], [_Prepared(p, b"k%d" % i, None, False, False) for i in range(9)],
                  [_Prepared(np.float32(1).reshape(()), b"z", None, False, False)],
                  [_Prepared(np.zeros((1,) * 17, np.float32), b"r", None, False, False)]):
        r2, k2 = _request("m", None, preps, N.ORDER_UPB, False)
        cap = C.c_uint64()
        assert lib.b200tfs_padded_request_arena_size(1, C.byref(r2), C.byref(cap)) in (N.E_ARG, N.E_DTYPE)
