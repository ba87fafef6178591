"""b200tfs_padded_request_frame_columns - the framing the padded encode's kernels write for one request with string columns, run on
the host from the same inline source - against the protobuf runtime's request of the request's boxes; the arena bound
b200tfs_padded_request_columns_arena_size against the protobuf sizes placed as the kernels place them; every refusal."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

import padded_strings_ref as R
import string_responses as SR
from min_tfs_client import _native as N
from tensorflow.core.framework import types_pb2

HERE = os.path.dirname(os.path.abspath(__file__))
DT_STRING, DT_FLOAT, DT_INT64, DT_BOOL = types_pb2.DT_STRING, types_pb2.DT_FLOAT, types_pb2.DT_INT64, types_pb2.DT_BOOL
_ENUM = {np.dtype(np.float32): DT_FLOAT, np.dtype(np.int64): DT_INT64, np.dtype(np.bool_): DT_BOOL}


class _Call:
    """The C structs of one request of the padded encode: padded / broadcast inputs, numeric arrays or string columns."""

    def __init__(self, padded, rows, broadcast, order=N.ORDER_UPB, grpc=False, version=3, name=b"model"):
        self.keys = list(padded) + list(broadcast)
        self.hold = []
        ts, pins, bs = [], [], []
        for k in self.keys:
            v = padded[k] if k in padded else broadcast[k]
            kb = k.encode()
            if isinstance(v, tuple):                    # (data, offsets, strings, dims)
                data, off, _, dims = v
                d = (C.c_int64 * max(len(dims), 1))(*dims)
                self.hold += [d, data, off]
                t = N.Tensor(data=data.ctypes.data if data.size else None, src_dtype=DT_STRING, wire_dtype=DT_STRING, rank=len(dims),
                             flags=N.F_DEVICE_DATA, dims=d, key=kb, key_len=len(kb), packed_len=0)
                bs.append(N.Bytes(offsets=off.ctypes.data, data_len=data.size, flags=N.F_DEVICE_DATA))
            else:
                a = np.ascontiguousarray(v)
                d = (C.c_int64 * max(a.ndim, 1))(*a.shape)
                self.hold += [d, a]
                t = N.Tensor(data=a.ctypes.data if a.size else None, src_dtype=_ENUM[a.dtype], wire_dtype=_ENUM[a.dtype], rank=a.ndim,
                             flags=N.F_DEVICE_DATA, dims=d, key=kb, key_len=len(kb), packed_len=0)
                bs.append(N.Bytes())
            if k in broadcast:
                t.flags |= N.F_BROADCAST
                pins.append(N.PadInput(shapes=None, cols=0))
            else:
                h = (C.c_int64 * len(rows[k]))(*[int(x) for x in rows[k]])
                self.hold.append(h)
                pins.append(N.PadInput(shapes=C.cast(h, C.c_void_p), cols=len(rows[k])))
            ts.append(t)
        self.ts = (N.Tensor * max(len(ts), 1))(*ts)
        self.pins = (N.PadInput * max(len(pins), 1))(*pins)
        self.bs = (N.Bytes * max(len(bs), 1))(*bs)
        self.req = N.Request(model_name=name, model_name_len=len(name), has_version=int(version is not None), order=order,
                             version=version or 0, n_inputs=len(ts), flags=N.RF_GRPC_FRAME if grpc else 0, inputs=self.ts)

    def frame(self, packed, cap=1 << 22):
        lib = N.load()
        n = len(self.keys)
        buf = np.full(cap, 0xEE, np.uint8)
        rl = C.c_uint64()
        qoff, qlen = (C.c_uint64 * max(n, 1))(), (C.c_uint64 * max(n, 1))()
        pk = (C.c_uint64 * max(n, 1))(*packed)
        rc = lib.b200tfs_padded_request_frame_columns(C.byref(self.req), self.pins, self.bs, pk, buf.ctypes.data, cap, C.byref(rl), qoff, qlen)
        return rc, buf, int(rl.value), [int(qoff[i]) for i in range(n)], [int(qlen[i]) for i in range(n)]


def _packed_varint(a) -> int:
    v = np.asarray(a).astype(np.int64).ravel().view(np.uint64)
    n = np.ones(v.shape, np.int64)
    for s in range(7, 64, 7):
        n += (v >> np.uint64(s)) != 0
    return int(n.sum())


def _check(padded, rows, broadcast, order="deterministic", grpc=False, version=3):
    """One request whose rows start at row 0 of each padded input, against the protobuf runtime."""
    pad_ref, bc_ref, packed = {}, {}, []
    for k in list(padded) + list(broadcast):
        v = padded[k] if k in padded else broadcast[k]
        (pad_ref if k in padded else bc_ref)[k] = (v[2], v[3]) if isinstance(v, tuple) else v
    ref = R.reference_requests("model", version, pad_ref, {k: [rows[k]] for k in padded}, bc_ref, order, grpc)[0]
    # the counted payloads: string_val values and packed varints of each box
    payloads = {}
    for k in list(padded) + list(broadcast):
        v = padded[k] if k in padded else broadcast[k]
        if isinstance(v, tuple):
            strs = R.box_strings(v[2], v[3], 0, rows[k])[0] if k in padded else v[2]
            payloads[k] = SR.strings_body(strs)
            packed.append(len(payloads[k]))
        else:
            box = v[(slice(0, int(rows[k][0])),) + tuple(slice(0, int(x)) for x in rows[k][1:])] if k in padded else v
            packed.append(_packed_varint(box) if v.dtype == np.int64 and box.size else 0)
    call = _Call(padded, rows, broadcast, N.ORDER_GIVEN if order == "given" else N.ORDER_UPB, grpc, version)
    rc, buf, rl, qoff, qlen = call.frame(packed)
    assert rc == N.OK, N.last_error()
    assert rl == len(ref)
    ref = np.frombuffer(ref, np.uint8)
    mask = np.ones(rl, bool)
    for i, k in enumerate(call.keys):
        mask[qoff[i]: qoff[i] + qlen[i]] = False
        assert (buf[qoff[i]: qoff[i] + qlen[i]] == 0xEE).all()          # payloads are the kernels'
        if k in payloads:                                                  # where the values go and how long they are
            assert ref[qoff[i]: qoff[i] + qlen[i]].tobytes() == payloads[k]
    assert (buf[:rl][mask] == ref[mask]).all()
    assert (buf[rl: rl + 64] == 0xEE).all()


def _col(rng, dims, max_len=40):
    data, off, strs = R.random_column(rng, dims, max_len)
    return data, off, strs, list(dims)


@pytest.mark.parametrize("rank", [1, 2, 3])
@pytest.mark.parametrize("trial", range(6))
def test_frame_matches_protobuf(rank, trial):
    rng = np.random.default_rng(rank * 31 + trial)
    dims = [int(rng.integers(1, 9))] + [int(rng.integers(0, 5)) for _ in range(rank - 1)]
    col = _col(rng, dims, max_len=[0, 3, 40, 200][trial % 4])
    full = trial % 2 == 1
    row = [int(rng.integers(0, dims[0] + 1))] + ([int(rng.integers(0, d + 1)) for d in dims[1:]] if full else [])
    padded = {"text": col, "ids": rng.integers(-(1 << 40), 1 << 40, (dims[0], 5)).astype(np.int64)}
    rows = {"text": row, "ids": [row[0], int(rng.integers(0, 6))]}
    bc = {"scale": np.float32([0.5, 2.0])}
    order = ["deterministic", "given"][trial % 2]
    _check(padded, rows, bc, order=order, grpc=trial % 3 == 0, version=None if trial == 5 else 9)


@pytest.mark.parametrize("rank", [0, 1, 2, 3])
def test_broadcast_strings(rank):
    rng = np.random.default_rng(100 + rank)
    dims = [int(rng.integers(0, 4)) for _ in range(rank)]
    _check({"x": np.arange(12, dtype=np.float32).reshape(4, 3)}, {"x": [2]}, {"image_bytes": _col(rng, dims, 300)})
    _check({"x": np.arange(12, dtype=np.float32).reshape(4, 3)}, {"x": [0, 0]}, {"image_bytes": _col(rng, dims, 0)}, order="given")


@pytest.mark.parametrize("axis", range(3))
def test_empty_boxes_and_zero_dims(axis):
    rng = np.random.default_rng(7 + axis)
    col = _col(rng, [5, 4, 3], 20)
    row = [3, 2, 2]
    row[axis] = 0
    _check({"s": col, "b": np.ones((5, 4), np.bool_)}, {"s": row, "b": [3, 4]}, {})


def test_long_strings_and_varint_edges():
    rng = np.random.default_rng(5)
    for n in (0, 127, 128, 16383, 16384, (1 << 21) - 1, 1 << 21):
        data = rng.integers(0, 256, n + 3).astype(np.uint8)
        off = np.array([0, n, n + 3], np.int64)
        strs = [data[:n].tobytes(), data[n:].tobytes()]
        _check({"s": (data, off, strs, [2])}, {"s": [2]}, {}, grpc=True)


def test_keys_in_both_orders_and_trimmed_dims():
    rng = np.random.default_rng(11)
    padded = {"zeta": _col(rng, [6, 5, 4], 9), "alpha": _col(rng, [6, 7], 9), "mid": rng.standard_normal((6, 3)).astype(np.float32)}
    rows = {"zeta": [4, 3, 2], "alpha": [4], "mid": [4, 2]}
    for order in ("deterministic", "given"):
        _check(padded, rows, {"b": _col(rng, [2], 5)}, order=order)


def _placed(lengths):
    at = 0
    for ln in lengths:
        at = ((at + 255) & ~255) + 127 + ln
    return at


def test_arena_size_bounds_protobuf_sizes():
    lib = N.load()
    rng = np.random.default_rng(3)
    for trial in range(12):
        n = int(rng.integers(1, 9))
        R_ = int(rng.integers(n, 3 * n + 1))
        dims = [R_, int(rng.integers(1, 5))]
        col = _col(rng, dims, [0, 5, 300][trial % 3])
        bcol = _col(rng, [int(rng.integers(0, 4))], 50)
        ids = rng.integers(-(1 << 62), 1 << 62, (R_, 3)).astype(np.int64)
        rows = np.zeros(n, np.int64)
        left = R_
        for r in range(n):
            rows[r] = int(rng.integers(0, left + 1)) if r < n - 1 else left
            left -= rows[r]
        S = np.stack([rows, rng.integers(0, dims[1] + 1, n)], axis=1)
        ref = R.reference_requests("m" * 40, 2 ** 40, {"s": (col[2], col[3]), "ids": ids}, {"s": S, "ids": rows}, {"b": (bcol[2], bcol[3])},
                                   grpc=True)
        call = _Call({"s": col, "ids": ids}, {"s": [1, 1], "ids": [1]}, {"b": bcol}, grpc=True, version=2 ** 40, name=b"m" * 40)
        cap = C.c_uint64()
        N.check(lib.b200tfs_padded_request_columns_arena_size(n, C.byref(call.req), call.bs, C.byref(cap)))
        assert cap.value >= _placed([len(w) for w in ref]) + 256


def test_refusals():
    lib = N.load()
    rng = np.random.default_rng(1)
    col = _col(rng, [4, 2], 5)
    buf = np.zeros(4096, np.uint8)
    rl = C.c_uint64()

    def codes(mutate):
        call = _Call({"s": col}, {"s": [2]}, {})
        mutate(call)
        cap = C.c_uint64()
        a = lib.b200tfs_padded_request_columns_arena_size(1, C.byref(call.req), call.bs, C.byref(cap))
        f = lib.b200tfs_padded_request_frame_columns(C.byref(call.req), call.pins, call.bs, None, buf.ctypes.data, buf.size, C.byref(rl),
                                                     None, None)
        g = lib.b200tfs_padded_request_frame(C.byref(call.req), call.pins, None, buf.ctypes.data, buf.size, C.byref(rl), None, None)
        return a, f, g

    assert codes(lambda c: None)[:2] == (N.OK, N.OK)
    assert codes(lambda c: None)[2] == N.E_DTYPE                          # DT_STRING without an entry (the plain entry point)

    def no_entry(c):
        c.bs[0] = N.Bytes()
    assert codes(no_entry)[:2] == (N.E_DTYPE, N.E_DTYPE)

    def other_dtype(c):
        c.ts[0].src_dtype = DT_FLOAT
    def other_wire(c):
        c.ts[0].wire_dtype = DT_FLOAT
    def content(c):
        c.ts[0].flags |= N.F_TENSOR_CONTENT
    def snan(c):
        c.ts[0].flags |= N.F_KEEP_SNAN
    def misaligned(c):
        c.bs[0].offsets += 4
    def negative(c):
        c.bs[0].data_len = -1
    def flags(c):
        c.bs[0].flags = 0x100
    for m in (other_dtype, other_wire, content, snan, misaligned, negative, flags):
        assert codes(m)[:2] == (N.E_ARG, N.E_ARG), m.__name__


def test_header_is_c99_and_symbols_exported():
    lib = N.load()
    for sym in ("b200tfs_padded_request_columns_arena_size", "b200tfs_encode_padded_requests_columns_async",
                "b200tfs_padded_request_frame_columns"):
        assert hasattr(lib, sym)
    cc = shutil.which(os.environ.get("CC") or "gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    out = subprocess.run([cc, "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-fsyntax-only",
                          os.path.join(HERE, "native", "abi_c99.c")], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr


def test_host_route_cuts_boxes_and_checks_only_their_offsets():
    """The host route's box of a padded column (calls the device route does not take) against the definition."""
    from min_tfs_client.codec import BytesColumn, _bytes_box
    rng = np.random.default_rng(21)
    for dims in [(7,), (6, 3), (5, 4, 3)]:
        data, off, strs = R.random_column(rng, list(dims), 9)
        col = BytesColumn(np.concatenate([np.zeros(2, np.uint8), data]), off + 2, dims)
        for t in range(20):
            r0 = int(rng.integers(0, dims[0] + 1))
            rows = int(rng.integers(0, dims[0] - r0 + 1))
            row = [rows] + ([int(rng.integers(0, d + 1)) for d in dims[1:]] if t % 2 else [])
            b = _bytes_box("k", col, r0, row)
            want, bd = R.box_strings(strs, dims, r0, row)
            assert [b.data[b.offsets[j]: b.offsets[j + 1]].tobytes() for j in range(len(want))] == want
            assert tuple(b.shape) == tuple(bd) and b.offsets.size == len(want) + 1
    o = np.arange(6, dtype=np.int64)
    o[4] = 0                                     # string 3 ends before it starts; string 4 starts before string 3 ends
    col = BytesColumn(np.zeros(5, np.uint8), o, (5,))
    assert _bytes_box("k", col, 0, [2]).offsets.tolist() == [0, 1, 2]
    with pytest.raises(ValueError):
        _bytes_box("k", col, 3, [2])
    assert _bytes_box("k", col, 4, [1]).offsets.tolist() == [0, 5]     # reads offsets 4, 4, 5, 5 only
