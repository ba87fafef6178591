"""Decode of a batch of PredictResponses with ragged trailing dims into one padded tensor per key (b200tfs_decode_padded), on three
workloads:

  P1  256 x {logits f32[1, T_r, 1024]}, T_r uniform in 32..512
  P2  1024 x {tokens int64[1, T_r] in 0..50 000, scores f32[1, T_r]}, T_r in 1..128
  P3  P1's shape at equal T (T = 272) - padded against b200tfs_decode_concat: what padding costs over concatenation

Legs (CUDA events around N calls after a warm-up, three runs each; the Python leg by the host clock):
  padded eager     b200tfs_decode_padded over a device arena
  padded graph     the same call captured once and replayed
  concat eager     b200tfs_decode_concat (P3 only)
  python           Codec.decode_predict_responses per response + numpy pad, host wire to host arrays
Every leg is compared bit for bit against the numpy definition after its timed region.  The card's name and power limit are
read and printed by the same command.

    python tools/padded_probe.py [--iters 20] [--workloads P1,P2,P3]
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
    if name == "P1":
        return [O.build_predict_response([("logits", rng.standard_normal((1, int(t), 1024), dtype=np.float32))])
                for t in rng.integers(32, 513, 256)]
    if name == "P2":
        return [O.build_predict_response([("tokens", rng.integers(0, 50001, (1, int(t)), dtype=np.int64)),
                                          ("scores", rng.standard_normal((1, int(t)), dtype=np.float32))])
                for t in rng.integers(1, 129, 1024)]
    return [O.build_predict_response([("logits", rng.standard_normal((1, 272, 1024), dtype=np.float32))]) for _ in range(256)]


def definition(codec, wires, keys):
    per = [codec.decode_predict_responses([w])[0][0] for w in wires]
    res = {}
    for k in keys:
        parts = [p[k] for p in per]
        tail = tuple(max(p.shape[d] for p in parts) for d in range(1, parts[0].ndim))
        a = np.full((sum(p.shape[0] for p in parts), *tail), 0, parts[0].dtype)
        r0 = 0
        for p in parts:
            a[(slice(r0, r0 + p.shape[0]),) + tuple(slice(0, d) for d in p.shape[1:])] = p
            r0 += p.shape[0]
        res[k] = a
    return res


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
    want = definition(codec, wires, keys)
    buf, off, ln = codec._pack_wires(wires)
    arena = codec.device_array(buf)
    nk = len(keys)
    pk = (N.PadKey * nk)()
    kb = [k.encode() for k in keys]
    for i, k in enumerate(kb):
        pk[i].key, pk[i].key_len = k, len(k)
    N.check(lib.b200tfs_padded_layout(buf.ctypes.data, n, off, ln, nk, pk, 0))
    dsts = []
    for i in range(nk):
        p = C.c_void_p()
        N.check(lib.b200tfs_malloc(ctx, max(int(pk[i].bytes), 16), C.byref(p)))
        dsts.append(p)
        pk[i].dst, pk[i].dst_cap = p.value, int(pk[i].bytes)
    outs, specs, st = (N.Output * (n * nk))(), (N.ModelSpec * n)(), (C.c_int32 * n)()

    def padded():
        N.check(lib.b200tfs_decode_padded(ctx, arena.ptr, n, off, ln, nk, pk))

    def check(label):
        N.check(lib.b200tfs_padded_results(ctx, n, nk, outs, specs, st))
        for i, k in enumerate(keys):
            h = np.empty(want[k].nbytes, np.uint8)
            N.check(lib.b200tfs_memcpy_d2h(ctx, h.ctypes.data, dsts[i].value, h.nbytes))
            N.check(lib.b200tfs_sync(ctx))
            assert h.tobytes() == want[k].tobytes(), (name, label, k)

    padded()
    check("warm-up")
    if name == "P3":          # size the concat decode's scratch before a captured graph pins the context's buffers
        ck = (N.ConcatKey * nk)()
        for i, k in enumerate(kb):
            ck[i].key, ck[i].key_len, ck[i].dst, ck[i].dst_cap = k, len(k), dsts[i].value, int(pk[i].bytes)
        N.check(lib.b200tfs_decode_concat(ctx, arena.ptr, n, off, ln, nk, ck))
        N.check(lib.b200tfs_sync(ctx))
    res = {"padded eager": timed(codec, padded, iters)}
    check("padded eager")
    gc_exec = C.c_void_p()
    N.check(lib.b200tfs_capture_begin(ctx))
    padded()
    N.check(lib.b200tfs_capture_end(ctx, C.byref(gc_exec)))
    N.check(lib.b200tfs_graph_launch(ctx, gc_exec))
    res["padded graph"] = timed(codec, lambda: N.check(lib.b200tfs_graph_launch(ctx, gc_exec)), iters)
    check("padded graph")
    N.check(lib.b200tfs_graph_destroy(gc_exec))
    if name == "P3":
        def concat():
            N.check(lib.b200tfs_decode_concat(ctx, arena.ptr, n, off, ln, nk, ck))
        concat()
        res["concat eager"] = timed(codec, concat, iters)
        N.check(lib.b200tfs_concat_results(ctx, n, nk, (N.Output * (n * nk))(), None, None))
        for i, k in enumerate(keys):
            h = np.empty(want[k].nbytes, np.uint8)
            N.check(lib.b200tfs_memcpy_d2h(ctx, h.ctypes.data, dsts[i].value, h.nbytes))
            N.check(lib.b200tfs_sync(ctx))
            assert h.tobytes() == want[k].tobytes(), (name, "concat", k)
    py = []
    for _ in range(3):
        t0 = time.perf_counter()
        got = definition(codec, wires, keys)
        py.append(1e6 * (time.perf_counter() - t0))
    assert all(got[k].tobytes() == want[k].tobytes() for k in keys)
    res["python"] = py
    out_bytes = sum(want[k].nbytes for k in keys)
    for d in dsts:
        lib.b200tfs_free(ctx, d)
    codec.close()
    return res, len(buf), out_bytes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--workloads", default="P1,P2,P3")
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                          text=True).stdout.strip()
    print(f"card: {card}")
    for name in a.workloads.split(","):
        res, wire, out = run(name, a.iters)
        print(f"{name}: wire {wire / 2**20:.1f} MiB, result {out / 2**20:.1f} MiB")
        for leg, us in res.items():
            print(f"  {leg:14s} " + " ".join(f"{u:10.1f}" for u in us) + " us/call")


if __name__ == "__main__":
    main()
