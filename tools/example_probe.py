"""Classify / Regress request encode on the GPU (b200tfs_encode_example_requests_*) against the host path it replaces.

Workloads (one request each unless stated):
  W1  65 536 examples x {dense f32[64]}                                   float-only: closed-form offsets, no count / scan
  W2  16 384 examples x {dense f32[64], ids int64[8] in 0..50 000, age f32}
  W3  256 requests of 64 examples shaped like W2
Legs: the _async entry point eager (device columns -> device arena), the same captured once as a CUDA graph and replayed,
_host from pinned columns (copies both ways included), and examples_from_input_dict + SerializeToString(deterministic=True)
on one host core.  CUDA events over >= 20 calls after warm-up, three runs each; bytes = column bytes read + wire bytes
written; the share is of the H100 SXM data sheet's 3.35 TB/s.  W1 is set beside the Predict encode (b200tfs_encode_requests_async)
of the same f32[65536, 64] as one tensor, and W2 is split by kernel with torch.profiler in a run of its own.  Every leg's
bytes are checked against the host path after its timed region.  Needs a GPU; --json PATH also writes every number there.

  python tools/example_probe.py [--calls 20] [--runs 3] [--json PATH]
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

from min_tfs_client import _native as N  # noqa: E402
from min_tfs_client.codec import Codec, _example_columns  # noqa: E402
from min_tfs_client.requests import TensorServingClient  # noqa: E402
from tensorflow_serving.apis.classification_pb2 import ClassificationRequest  # noqa: E402

PEAK = 3.35e12


def workloads(rng):
    def w2(n):
        return {"dense": rng.standard_normal((n, 64)).astype(np.float32), "ids": rng.integers(0, 50_000, (n, 8)),
                "age": rng.standard_normal(n).astype(np.float32)}
    return {"W1": [{"dense": rng.standard_normal((65536, 64)).astype(np.float32)}], "W2": [w2(16384)], "W3": [w2(64) for _ in range(256)]}


def host_ref(d):
    return TensorServingClient._make_example_request(None, ClassificationRequest, "model", d, 1).SerializeToString(deterministic=True)


class Ctx:
    def __init__(self):
        self.lib = N.load()
        self.ctx = C.c_void_p()
        N.check(self.lib.b200tfs_create(0, C.byref(self.ctx)))
        self.ev = [C.c_void_p(), C.c_void_p()]
        for e in self.ev:
            N.check(self.lib.b200tfs_event_create(C.byref(e)))

    def malloc(self, nb):
        p = C.c_void_p()
        N.check(self.lib.b200tfs_malloc(self.ctx, max(int(nb), 1), C.byref(p)))
        return p.value

    def timed(self, fn, calls):
        N.check(self.lib.b200tfs_event_record(self.ctx, self.ev[0]))
        for _ in range(calls):
            fn()
        N.check(self.lib.b200tfs_event_record(self.ctx, self.ev[1]))
        N.check(self.lib.b200tfs_event_sync(self.ev[1]))
        ms = C.c_float()
        N.check(self.lib.b200tfs_event_elapsed_ms(self.ev[0], self.ev[1], C.byref(ms)))
        return ms.value * 1e3 / calls


def timed_host(fn, calls):
    """a synchronous call: the host clock around it is the call's time"""
    t0 = time.perf_counter()
    for _ in range(calls):
        fn()
    return (time.perf_counter() - t0) * 1e6 / calls


def build(dicts, device_ptrs=None):
    keep, structs = [], []
    for r, d in enumerate(dicts):
        n, preps = _example_columns(d)
        feats = (N.Feature * len(preps))(*[p[0] for p in preps])
        if device_ptrs is not None:
            for k, f in enumerate(feats):
                f.data = device_ptrs[r][k]
                f.flags |= N.F_DEVICE_DATA
        structs.append(N.ExampleRequest(model_name=b"model", model_name_len=5, has_version=1, order=N.ORDER_UPB, version=1,
                                        n_examples=n, n_features=len(preps), flags=0, features=feats))
        keep.append((preps, feats))
    return (N.ExampleRequest * len(structs))(*structs), keep


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--json", metavar="PATH", help="write every number of the run to PATH as JSON")
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    rng = np.random.default_rng(0)
    W = workloads(rng)
    lib = N.load()
    codec = Codec(0)
    out = {"card": card, "calls": args.calls, "runs": args.runs, "workloads": {}}
    for name, dicts in W.items():
        g = Ctx()       # a context per workload: the graph captured below pins its scratch buffers
        refs = [host_ref(d) for d in dicts]
        col_bytes = sum(a.nbytes for d in dicts for a in d.values())
        wire_bytes = sum(len(w) for w in refs)
        moved = col_bytes + wire_bytes
        # device columns
        ptrs = []
        for d in dicts:
            row = []
            for a in d.values():
                p = g.malloc(a.nbytes)
                N.check(lib.b200tfs_memcpy_h2d(g.ctx, p, a.ctypes.data, a.nbytes))
                row.append(p)
            ptrs.append(row)
        reqs, keep = build(dicts, ptrs)
        n = len(dicts)
        cap = C.c_uint64()
        N.check(lib.b200tfs_example_arena_size(n, reqs, C.byref(cap)))
        arena = g.malloc(cap.value)
        off, ln = (C.c_uint64 * n)(), (C.c_uint64 * n)()

        def eager():
            N.check(lib.b200tfs_encode_example_requests_async(g.ctx, n, reqs, arena, cap.value))

        def check_arena():
            N.check(lib.b200tfs_encode_results(g.ctx, n, off, ln))
            for i in range(n):
                buf = np.empty(ln[i], np.uint8)
                N.check(lib.b200tfs_memcpy_d2h(g.ctx, buf.ctypes.data, arena + off[i], ln[i]))
                N.check(lib.b200tfs_sync(g.ctx))
                assert buf.tobytes() == refs[i], (name, i)

        res = {"column_bytes": col_bytes, "wire_bytes": wire_bytes}
        for _ in range(3):
            eager()
        N.check(lib.b200tfs_sync(g.ctx))
        res["async_us"] = [g.timed(eager, args.calls) for _ in range(args.runs)]
        check_arena()
        N.check(lib.b200tfs_capture_begin(g.ctx))
        eager()
        ge = C.c_void_p()
        N.check(lib.b200tfs_capture_end(g.ctx, C.byref(ge)))
        launch = lambda: N.check(lib.b200tfs_graph_launch(g.ctx, ge))  # noqa: E731
        for _ in range(3):
            launch()
        res["graph_us"] = [g.timed(launch, args.calls) for _ in range(args.runs)]
        check_arena()
        N.check(lib.b200tfs_graph_destroy(ge))
        # _host from pinned columns (another context: the graph above pins this one's scratch buffers)
        pinned = [{k: codec.pinned_empty(a.shape, a.dtype) for k, a in d.items()} for d in dicts]
        for p, d in zip(pinned, dicts):
            for k in d:
                p[k][...] = d[k]
        hreqs, hkeep = build(pinned)
        wire = N.PinnedBuffer(cap.value)
        hoff, hln = (C.c_uint64 * n)(), (C.c_uint64 * n)()
        host = lambda: N.check(lib.b200tfs_encode_example_requests_host(codec.ctx, n, hreqs, wire.ptr, cap.value, hoff, hln))  # noqa: E731
        for _ in range(3):
            host()
        res["host_pinned_us"] = [timed_host(host, args.calls) for _ in range(args.runs)]
        assert all(wire.array[hoff[i]: hoff[i] + hln[i]].tobytes() == refs[i] for i in range(n)), name
        # the host path it replaces, one core
        runs = []
        for _ in range(args.runs):
            t0 = time.perf_counter()
            for d in dicts:
                host_ref(d)
            runs.append((time.perf_counter() - t0) * 1e6)
        res["protobuf_host_us"] = runs
        for leg in ("async_us", "graph_us", "host_pinned_us", "protobuf_host_us"):
            best = min(res[leg])
            res[leg.replace("_us", "_GBps")] = moved / best / 1e3
            res[leg.replace("_us", "_of_peak")] = moved / best / 1e-6 / PEAK
        out["workloads"][name] = res
        print(name, json.dumps({k: v for k, v in res.items()}), flush=True)
        if name == "W1":     # the Predict encode of the same bytes, one tensor
            a = dicts[0]["dense"]
            dims = (C.c_int64 * 2)(*a.shape)
            t = N.Tensor(data=ptrs[0][0], src_dtype=1, wire_dtype=1, rank=2, flags=0, dims=dims, key=b"dense", key_len=5,
                         packed_len=0)
            pr = N.Request(model_name=b"model", model_name_len=5, has_version=1, order=N.ORDER_UPB, version=1, n_inputs=1, flags=0,
                           inputs=C.pointer(t))
            pcap = C.c_uint64()
            N.check(lib.b200tfs_request_arena_size(1, C.byref(pr), C.byref(pcap)))
            parena = g.malloc(pcap.value + 4096)     # the async route's slot: the record's worst case + alignment
            pe = lambda: N.check(lib.b200tfs_encode_requests_async(g.ctx, 1, C.byref(pr), parena, pcap.value + 4096))  # noqa: E731
            for _ in range(3):
                pe()
            out["predict_same_bytes_async_us"] = [g.timed(pe, args.calls) for _ in range(args.runs)]
            print("predict W1-bytes", out["predict_same_bytes_async_us"], flush=True)
        if name == "W2":     # per-kernel split, profiler on, in a run of its own
            import torch
            from torch.profiler import ProfilerActivity, profile

            torch.cuda.init()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.calls):
                    eager()
                N.check(lib.b200tfs_sync(g.ctx))
            split = {}
            for e in prof.key_averages():
                if "ex_" in e.key:
                    total = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
                    split[e.key] = {"count": e.count, "avg_us": total / max(e.count, 1)}
            out["W2_kernels"] = split
            print("W2 kernels", json.dumps(split), flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)
    codec.close()


if __name__ == "__main__":
    main()
