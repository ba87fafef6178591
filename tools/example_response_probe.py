"""Classify / Regress response decode on the GPU (b200tfs_decode_example_responses*) against the host path it replaces.

Workloads:
  R1  1 response x 65 536 regressions
  R2  256 responses x 64 examples, C = 2, labels "0" / "1"
  R3  64 responses x 64 examples x 1000 labelled classes, the same labels in every example
  R4  R3's shape with C = 5 and labels that differ per example
Legs: the _async entry point eager and as a replayed CUDA graph (device wire -> device values; CUDA events over --calls calls
after warm-up, --runs runs); _host_async + results from a pinned wire (host clock around synchronised calls); the Python call
Codec.decode_*_responses end to end (host clock); FromString + extraction on one host core.  GB/s counts wire bytes read plus
values (and label references) written.  Every leg's output is compared bitwise with the host path after its timed region.
--profile splits R1 and R3 by kernel with torch.profiler (run it on its own).  Needs a GPU; --json PATH writes every number.

  python tools/example_response_probe.py [--calls 20] [--runs 3] [--json PATH] [--profile]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "min-tfs-client_b200"))
sys.path.insert(0, os.path.join(REPO, "tests"))

import example_response_corpus as X  # noqa: E402
from min_tfs_client import _native as N  # noqa: E402
from min_tfs_client.codec import Codec  # noqa: E402


def workloads(rng):
    return {
        "R1": (X.REGRESS, [X.random_regression(rng, 65536)]),
        "R2": (X.CLASSIFY, [X.random_classification(rng, 64, ["0", "1"]) for _ in range(256)]),
        "R3": (X.CLASSIFY, [X.random_classification(rng, 64, [f"class_{k:04d}" for k in range(1000)]) for _ in range(64)]),
        "R4": (X.CLASSIFY, [X.random_classification(rng, 64, lambda i: [f"label_{(i * 31 + k * 7) % 1000}" for k in range(5)])
                            for _ in range(64)]),
    }


def host_decode(kind, wires):
    """FromString + extraction: what a client of the reference runs."""
    vals, labels, _ = X.expected(kind, wires)
    return vals, labels


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--json", metavar="PATH")
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    lib = N.load()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print("gpu:", gpu, flush=True)
    out = {"gpu": gpu}
    ev = [C.c_void_p(), C.c_void_p()]
    for e in ev:
        N.check(lib.b200tfs_event_create(C.byref(e)))

    def malloc(nb):
        p = C.c_void_p()
        N.check(lib.b200tfs_malloc(ctx, max(int(nb), 1), C.byref(p)))
        held.append(p.value)
        return p.value

    rng = np.random.default_rng(20261016)
    codec = Codec(0)
    for name, (kind, wires) in workloads(rng).items():
        ctx, held = C.c_void_p(), []          # a context per workload: a captured graph pins its scratch buffers
        N.check(lib.b200tfs_create(0, C.byref(ctx)))
        n = len(wires)
        lens = [len(w) for w in wires]
        offs = np.cumsum([0] + [(x + 255) & ~255 for x in lens[:-1]]).astype(np.uint64)
        total = int(offs[-1]) + lens[-1]
        pin = N.PinnedBuffer(total + 256)
        for o, w in zip(offs, wires):
            pin.array[int(o): int(o) + len(w)] = np.frombuffer(w, np.uint8)
        off, ln = (C.c_uint64 * n)(*offs.tolist()), (C.c_uint64 * n)(*lens)
        arena = malloc(total + 256)
        N.check(lib.b200tfs_memcpy_h2d(ctx, arena, pin.ptr, total))
        mr, mv = C.c_uint64(), C.c_uint64()
        N.check(lib.b200tfs_example_response_bound(kind, n, ln, C.byref(mr), C.byref(mv)))
        vdst, ldst = malloc(4 * mv.value), malloc(8 * mv.value) if kind == X.CLASSIFY else None
        lcap = mv.value if kind == X.CLASSIFY else 0
        per, specs, batch = (C.c_int64 * (3 * n))(), (N.ModelSpec * n)(), (C.c_int64 * 5)()
        t0 = time.perf_counter()
        ref_vals, ref_labels = host_decode(kind, wires)
        host_s = time.perf_counter() - t0
        rows = int(ref_vals.shape[0])
        moved = sum(lens) + ref_vals.nbytes + (8 * ref_vals.size if kind == X.CLASSIFY else 0)
        res = {"wire_bytes": sum(lens), "rows": rows, "host_fromstring_ms": host_s * 1e3}

        def call():
            N.check(lib.b200tfs_decode_example_responses(ctx, kind, arena, n, off, ln, vdst, mv.value, ldst, lcap))

        def verify(tag):
            N.check(lib.b200tfs_example_response_results(ctx, n, per, specs, batch))
            assert batch[3] == N.OK and batch[0] == rows, (tag, list(batch))
            got = np.empty(ref_vals.size, np.float32)
            if got.nbytes:
                N.check(lib.b200tfs_memcpy_d2h(ctx, got.ctypes.data, vdst, got.nbytes))
                N.check(lib.b200tfs_sync(ctx))
            assert np.array_equal(got.view(np.uint32), np.ascontiguousarray(ref_vals).ravel().view(np.uint32)), tag

        def timed(fn, label):
            best = []
            for _ in range(args.runs):
                N.check(lib.b200tfs_event_record(ctx, ev[0]))
                for _ in range(args.calls):
                    fn()
                N.check(lib.b200tfs_event_record(ctx, ev[1]))
                N.check(lib.b200tfs_event_sync(ev[1]))
                ms = C.c_float()
                N.check(lib.b200tfs_event_elapsed_ms(ev[0], ev[1], C.byref(ms)))
                best.append(ms.value / args.calls)
            res[label + "_us"] = [round(1e3 * b, 2) for b in best]
            res[label + "_gbs"] = round(moved / (min(best) * 1e-3) / 1e9, 2)

        for _ in range(3):
            call()
        verify("warm-up")
        timed(call, "async_eager")
        verify("async_eager")
        def host_async():
            N.check(lib.b200tfs_decode_example_responses_host_async(ctx, kind, pin.ptr, n, off, ln, vdst, mv.value, ldst, lcap))
            N.check(lib.b200tfs_example_response_results(ctx, n, per, specs, batch))

        host_async()                          # sizes the staging buffer before the capture pins it
        call()
        N.check(lib.b200tfs_capture_begin(ctx))
        call()
        g = C.c_void_p()
        N.check(lib.b200tfs_capture_end(ctx, C.byref(g)))
        timed(lambda: N.check(lib.b200tfs_graph_launch(ctx, g)), "graph")
        verify("graph")
        N.check(lib.b200tfs_graph_destroy(g))

        for label, fn in (("host_async_results", host_async),
                          ("python_call", lambda: (codec.decode_regression_responses if kind == X.REGRESS
                                                   else codec.decode_classification_responses)(wires))):
            fn()
            ts = []
            for _ in range(args.runs):
                t0 = time.perf_counter()
                for _ in range(args.calls):
                    r = fn()
                ts.append((time.perf_counter() - t0) / args.calls)
            res[label + "_us"] = [round(1e6 * t, 1) for t in ts]
            res[label + "_gbs"] = round(moved / min(ts) / 1e9, 2)
        verify("host_async")
        vals = r.values if kind == X.REGRESS else r.scores
        assert np.array_equal(np.ascontiguousarray(vals).view(np.uint32), np.ascontiguousarray(ref_vals).view(np.uint32))
        if kind == X.CLASSIFY:
            assert r.labels() == ref_labels
            res["same_labels"] = r.class_labels is not None
        print(name, json.dumps(res), flush=True)
        out[name] = res
        if args.profile and name in ("R1", "R3"):
            import torch
            from torch.profiler import ProfilerActivity, profile

            torch.cuda.init()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.calls):
                    call()
                N.check(lib.b200tfs_sync(ctx))
            split = {}
            for e in prof.key_averages():
                if "xr_" in e.key:
                    k = e.key.split("(")[0].split("::")[-1].replace("void ", "")
                    split[k] = round(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0)) / args.calls, 2)
            print(name, "kernels_us", json.dumps(split), flush=True)
            out[name + "_kernels_us"] = split
        pin.free()
        for p in held:
            lib.b200tfs_free(ctx, p)
        lib.b200tfs_destroy(ctx)
    codec.close()
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
