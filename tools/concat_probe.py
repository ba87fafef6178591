"""Decode of a batch of PredictResponses into one tensor per key (b200tfs_decode_concat) against the slot decode and the
Python route, on three workloads:

  A  256 x {scores f32[32,1000]}
  B  256 x {classes int64[32,5] (0..999), scores f32[32,5]}
  C  256 x {x f32[1024,1024]}  (a 1 GiB result)

Legs (CUDA events around N calls after a warm-up, three runs each; the Python leg by the host clock):
  concat eager     b200tfs_decode_concat over a device arena
  concat graph     the same call captured once and replayed
  slot decode      b200tfs_decode_responses of the same batch (record i into slot i)
  python           Codec.decode_predict_responses + np.concatenate, host wire to host arrays

    python tools/concat_probe.py [--iters 20] [--workloads ABC]
"""
import argparse
import ctypes as C
import os
import subprocess
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(REPO, "min-tfs-client_b200"), REPO]

from min_tfs_client import _native as N  # noqa: E402
from min_tfs_client.codec import Codec  # noqa: E402
from oracle import wire_oracle as O  # noqa: E402


def workload(name):
    rng = np.random.default_rng(0)
    if name == "A":
        return [O.build_predict_response([("scores", rng.standard_normal((32, 1000), dtype=np.float32))]) for _ in range(256)]
    if name == "B":
        return [O.build_predict_response([("classes", rng.integers(0, 1000, (32, 5), dtype=np.int64)),
                                          ("scores", rng.standard_normal((32, 5), dtype=np.float32))]) for _ in range(256)]
    x = rng.standard_normal((1024, 1024), dtype=np.float32)
    return [O.build_predict_response([("x", x)]) for _ in range(256)]


def timed(codec, fn, iters):
    lib, ctx = codec._lib, codec.ctx
    a, b = C.c_void_p(), C.c_void_p()
    N.check(lib.b200tfs_event_create(C.byref(a)))
    N.check(lib.b200tfs_event_create(C.byref(b)))
    out = []
    for _ in range(3):
        N.check(lib.b200tfs_event_record(ctx, a))
        for _ in range(iters):
            fn()
        N.check(lib.b200tfs_event_record(ctx, b))
        N.check(lib.b200tfs_event_sync(b))
        ms = C.c_float()
        N.check(lib.b200tfs_event_elapsed_ms(a, b, C.byref(ms)))
        out.append(1000.0 * ms.value / iters)
    lib.b200tfs_event_destroy(a)
    lib.b200tfs_event_destroy(b)
    return out


def run(name, iters):
    wires = workload(name)
    n = len(wires)
    keys = list(O.decode_predict_response(wires[0]))
    codec = Codec(0)
    lib, ctx = codec._lib, codec.ctx
    buf, off, ln = codec._pack_wires(wires)
    arena = codec.device_array(buf)
    nk = len(keys)
    ck = (N.ConcatKey * nk)()
    kb = [k.encode() for k in keys]
    for i, k in enumerate(kb):
        ck[i].key, ck[i].key_len = k, len(k)
    N.check(lib.b200tfs_concat_layout(buf.ctypes.data, n, off, ln, nk, ck, 0))
    dsts = []
    for i in range(nk):
        p = C.c_void_p()
        N.check(lib.b200tfs_malloc(ctx, max(int(ck[i].bytes), 1), C.byref(p)))
        dsts.append(p)
        ck[i].dst, ck[i].dst_cap = p.value, int(ck[i].bytes)
    payload = sum(int(ck[i].bytes) for i in range(nk))
    eager = lambda: N.check(lib.b200tfs_decode_concat(ctx, arena.ptr, n, off, ln, nk, ck))  # noqa: E731
    for _ in range(3):
        eager()
    outs, st = (N.Output * (n * nk))(), (C.c_int32 * n)()
    N.check(lib.b200tfs_concat_results(ctx, n, nk, outs, None, st))
    assert all(outs[j].status == N.OK for j in range(n * nk)), "the batch did not take the device route"
    want = {k: np.concatenate([O.decode_predict_response(w)[k] for w in wires[:8]]) for k in keys}
    for i, k in enumerate(keys):
        got = np.empty(want[k].nbytes, np.uint8)
        N.check(lib.b200tfs_memcpy_d2h(ctx, got.ctypes.data, dsts[i], got.nbytes))
        codec.sync()
        assert got.tobytes() == want[k].tobytes(), k
    t_eager = timed(codec, eager, iters)
    # graph: a context of its own (a captured graph pins the scratch buffers)
    gcodec = Codec(0)
    glib, gctx = gcodec._lib, gcodec.ctx
    gcall = lambda: N.check(glib.b200tfs_decode_concat(gctx, arena.ptr, n, off, ln, nk, ck))  # noqa: E731
    gcall()
    gcodec.sync()
    N.check(glib.b200tfs_capture_begin(gctx))
    gcall()
    g = C.c_void_p()
    N.check(glib.b200tfs_capture_end(gctx, C.byref(g)))
    for _ in range(3):
        N.check(glib.b200tfs_graph_launch(gctx, g))
    t_graph = timed(gcodec, lambda: N.check(glib.b200tfs_graph_launch(gctx, g)), iters)
    N.check(glib.b200tfs_graph_destroy(g))
    # the slot decode of the same batch
    need = C.c_uint64()
    N.check(lib.b200tfs_decode_slot_bytes(buf.ctypes.data, n, off, ln, 1, C.byref(need), None))
    stride = (max(int(need.value), max(int(x) for x in ln) + 256 * 9) + 255) & ~255
    varints = any(np.dtype(v.dtype).kind in "iub" for v in want.values())
    slot = C.c_void_p()
    N.check(lib.b200tfs_malloc(ctx, stride * n, C.byref(slot)))
    N.check(lib.b200tfs_set_decode_varints(ctx, 1 if varints else 0))
    sdec = lambda: N.check(lib.b200tfs_decode_responses(ctx, arena.ptr, n, off, ln, slot.value, stride))  # noqa: E731
    for _ in range(3):
        sdec()
    t_slot = timed(codec, sdec, iters)
    N.check(lib.b200tfs_set_decode_varints(ctx, 0))
    # Python: the per-response route and a concatenate on the host
    py = []
    for _ in range(3):
        t0 = time.perf_counter()
        res = codec.decode_predict_responses(wires)
        cat = {k: np.concatenate([r[0][k] for r in res]) for k in keys}
        py.append(1e6 * (time.perf_counter() - t0))
        del res, cat
    t1 = time.perf_counter()
    codec.decode_predict_responses_concat(wires, keys)
    py_concat = 1e6 * (time.perf_counter() - t1)
    for p in dsts + [slot]:
        lib.b200tfs_free(ctx, p)
    gcodec.close()
    codec.close()
    fmt = lambda xs: " / ".join(f"{x:.1f}" for x in xs)  # noqa: E731
    gbs = lambda us: 2 * payload / (us * 1e-6) / 1e9  # noqa: E731
    print(f"{name}: {n} records, {payload / 2**20:.2f} MiB decoded")
    print(f"  concat eager   us/call {fmt(t_eager)}   ({gbs(min(t_eager)):.0f} GB/s of 2P)")
    print(f"  concat graph   us/call {fmt(t_graph)}   ({gbs(min(t_graph)):.0f} GB/s of 2P)")
    print(f"  slot decode    us/call {fmt(t_slot)}   ({gbs(min(t_slot)):.0f} GB/s of 2P)")
    print(f"  python + np.concatenate  us {fmt(py)}   (decode_predict_responses_concat, host in and out: {py_concat:.0f} us)")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--workloads", default="ABC")
    args = ap.parse_args()
    try:
        print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv"], capture_output=True, text=True).stdout.strip())
    except OSError:
        print("nvidia-smi not found")
    for w in args.workloads:
        run(w, args.iters)


if __name__ == "__main__":
    main()
