#!/usr/bin/env python
"""Throughput of the batched / varint paths on one GPU (numbers for DESIGN.md; not the bench line).

    python tools/batch_probe.py            # prints one JSON object
"""
import ctypes as C
import json
import os
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(REPO, "min-tfs-client_b200"), os.path.join(REPO, "tests"), REPO]
from devutil import Dev  # noqa: E402
from min_tfs_client import _native as N  # noqa: E402


def timed(dev, fn, reps):
    lib = dev.lib
    e0, e1 = C.c_void_p(), C.c_void_p()
    N.check(lib.b200tfs_event_create(C.byref(e0)))
    N.check(lib.b200tfs_event_create(C.byref(e1)))
    fn()
    dev.sync()
    t0 = time.perf_counter()
    N.check(lib.b200tfs_event_record(dev.ctx, e0))
    for _ in range(reps):
        fn()
    N.check(lib.b200tfs_event_record(dev.ctx, e1))
    N.check(lib.b200tfs_event_sync(e1))
    wall = (time.perf_counter() - t0) / reps
    ms = C.c_float()
    N.check(lib.b200tfs_event_elapsed_ms(e0, e1, C.byref(ms)))
    return ms.value / reps * 1e-3, wall


def main():
    dev = Dev(0)
    lib = dev.lib
    out = {}
    peak = json.load(open(os.path.join(REPO, "MEASURED_PEAKS.json")))["hbm_gbs"] if os.path.exists(os.path.join(REPO, "MEASURED_PEAKS.json")) else 3350.0
    # ---- C5 share: 1024 x fp32[3,224,224] ------------------------------------------------------
    n, P = 1024, 3 * 224 * 224 * 4
    src = dev.malloc(n * P)
    N.check(lib.b200tfs_memset(dev.ctx, src, 0x3C, n * P))
    dims = (C.c_int64 * 3)(3, 224, 224)
    ts, rq = (N.Tensor * n)(), (N.Request * n)()
    for i in range(n):
        ts[i] = N.Tensor(data=src + i * P, src_dtype=1, wire_dtype=1, rank=3, flags=0, dims=dims, key=b"image", key_len=5, packed_len=0)
        rq[i] = N.Request(model_name=b"default", model_name_len=7, has_version=1, order=N.ORDER_UPB, version=1, n_inputs=1, flags=0,
                          inputs=C.cast(C.byref(ts, i * C.sizeof(N.Tensor)), C.POINTER(N.Tensor)))
    need = C.c_uint64()
    N.check(lib.b200tfs_request_arena_size(n, rq, C.byref(need)))
    arena = dev.malloc(need.value)
    off, ln = (C.c_uint64 * n)(), (C.c_uint64 * n)()
    enc = lambda: N.check(lib.b200tfs_encode_requests(dev.ctx, n, rq, arena, need.value, off, ln))  # noqa: E731
    t, wall = timed(dev, enc, 10)
    alg = n * (2 * P + 52)
    out["c5_encode_1024x602KB"] = {"gpu_ms": t * 1e3, "host_ms_per_call": wall * 1e3, "algorithmic_GBs": alg / t / 1e9, "frac_of_peak": alg / t / 1e9 / peak}
    # decode the same amount: responses laid out by hand (header + payload + model_spec)
    sys.path.insert(0, REPO)
    from oracle import wire_oracle
    one = wire_oracle.build_predict_response([("image", np.zeros((3, 224, 224), np.float32))])
    stride = (len(one) + 255) & ~255
    wire = dev.malloc(stride * n)
    host = np.zeros(stride * n, np.uint8)
    for i in range(n):
        host[i * stride: i * stride + len(one)] = np.frombuffer(one, np.uint8)
    N.check(lib.b200tfs_memcpy_h2d(dev.ctx, wire, host.ctypes.data, host.size))
    roff = (C.c_uint64 * n)(*[i * stride for i in range(n)])
    rlen = (C.c_uint64 * n)(*[len(one)] * n)
    dst_stride = (P + 255) & ~255
    dst = dev.malloc(dst_stride * n)
    dec = lambda: N.check(lib.b200tfs_decode_responses(dev.ctx, wire, n, roff, rlen, dst, dst_stride))  # noqa: E731
    t, wall = timed(dev, dec, 10)
    alg = n * (2 * P + len(one) - P)
    out["c5_decode_1024x602KB"] = {"gpu_ms": t * 1e3, "host_ms_per_call": wall * 1e3, "algorithmic_GBs": alg / t / 1e9, "frac_of_peak": alg / t / 1e9 / peak}
    # ---- varint: int64 [16M] with mixed magnitudes ---------------------------------------------
    m = 16 << 20
    rng = np.random.default_rng(0)
    vals = (rng.integers(0, 2 ** 62, size=m, dtype=np.int64) >> rng.integers(0, 62, size=m)).astype(np.int64)
    vals[::7] *= -1
    v = dev.upload(vals)
    vd = (C.c_int64 * 1)(m)
    vt = (N.Tensor * 1)(N.Tensor(data=v, src_dtype=9, wire_dtype=9, rank=1, flags=0, dims=vd, key=b"", key_len=0, packed_len=0))
    N.check(lib.b200tfs_measure(dev.ctx, 1, vt))
    packed = int(vt[0].packed_len)
    need2 = C.c_uint64()
    N.check(lib.b200tfs_tensor_arena_size(1, vt, C.byref(need2)))
    arena2 = dev.malloc(need2.value)
    o2, l2 = (C.c_uint64 * 1)(), (C.c_uint64 * 1)()
    venc = lambda: N.check(lib.b200tfs_encode_tensor_protos(dev.ctx, 1, vt, arena2, need2.value, o2, l2))  # noqa: E731
    t, wall = timed(dev, venc, 5)
    out["varint_encode_int64_16M"] = {"gpu_ms": t * 1e3, "payload_GBs": m * 8 / t / 1e9, "packed_bytes": packed,
                                      "algorithmic_GBs": (m * 8 + packed) / t / 1e9, "frac_of_peak": (m * 8 + packed) / t / 1e9 / peak}
    tm, _ = timed(dev, lambda: N.check(lib.b200tfs_measure(dev.ctx, 1, vt)), 5)
    out["varint_measure_int64_16M"] = {"gpu_ms": tm * 1e3, "payload_GBs": m * 8 / tm / 1e9}
    outs = (N.Output * 1)()
    st = (C.c_int32 * 1)()
    N.check(lib.b200tfs_parse_tensor_protos(dev.ctx, arena2, 1, o2, l2, outs, st))
    assert st[0] == 0 and outs[0].n_elems == m
    back = dev.malloc(m * 8)
    dptr = (C.c_void_p * 1)(back)
    vdec = lambda: N.check(lib.b200tfs_unpack_outputs(dev.ctx, arena2, 1, outs, o2, dptr, None, None))  # noqa: E731
    t, wall = timed(dev, vdec, 5)
    out["varint_decode_int64_16M"] = {"gpu_ms": t * 1e3, "payload_GBs": m * 8 / t / 1e9, "algorithmic_GBs": (m * 8 + packed) / t / 1e9,
                                      "frac_of_peak": (m * 8 + packed) / t / 1e9 / peak}
    assert np.array_equal(dev.download(back, m * 8).view(np.int64), vals)
    print(json.dumps(out, indent=1))
    dev.close()


if __name__ == "__main__":
    main()
