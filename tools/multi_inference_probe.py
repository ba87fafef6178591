"""MultiInference on the GPU: the response decode (b200tfs_decode_multi_inference_responses) against the Classify decode plus the
Regress decode of the same results, and the request encode (b200tfs_encode_example_tasks_async) against the same columns without
tasks.

Workloads:
  MI1  256 responses x 64 examples x {classify C = 2, regress}
  MI2  64 responses x 1000 examples x {classify C = 2, regress, classify C = 2}
  E2   256 requests of 64 examples x {f32[16], i64[4]} (W2-shaped) with two tasks, against the same requests without tasks
Every leg runs eager and as a replayed CUDA graph: CUDA events around --calls calls after a warm-up, --runs runs (the minimum
and the median of the per-call times are reported).  Each leg's output is compared bit for bit with protobuf after its timed
region.  Needs a GPU; --json PATH writes every number.

  python tools/multi_inference_probe.py [--calls 20] [--runs 3] [--json PATH]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "min-tfs-client_b200"))
sys.path.insert(0, os.path.join(REPO, "tests"))

import multi_inference_corpus as M  # noqa: E402
from min_tfs_client import _native as N  # noqa: E402
from min_tfs_client.codec import get_codec  # noqa: E402
from min_tfs_client.requests import CLASSIFY_METHOD_NAME, REGRESS_METHOD_NAME, make_multi_inference_request  # noqa: E402


class Timer:
    def __init__(self, lib, ctx):
        import torch
        self.torch, self.lib, self.ctx = torch, lib, ctx

    def run(self, fn, calls, runs):
        """per-call microseconds of `runs` runs of `calls` calls (CUDA events on the codec's stream)"""
        t = self.torch
        out = []
        fn()
        N.check(self.lib.b200tfs_sync(self.ctx))
        for _ in range(runs):
            N.check(self.lib.b200tfs_sync(self.ctx))
            a, b = t.cuda.Event(enable_timing=True), t.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(calls):
                fn()
            N.check(self.lib.b200tfs_sync(self.ctx))
            b.record()
            b.synchronize()
            out.append(1000.0 * a.elapsed_time(b) / calls)
        return out


_CODECS = []


def fresh():
    """the context of a new Codec (kept alive for the run)"""
    from min_tfs_client.codec import Codec
    _CODECS.append(Codec())
    return _CODECS[-1].ctx


def stage(lib, ctx, wires):
    blob = b"".join(w.ljust((len(w) + 255) & ~255, b"\0") for w in wires)
    offs = np.cumsum([0] + [(len(w) + 255) & ~255 for w in wires[:-1]]).astype(np.uint64)
    arena = C.c_void_p()
    N.check(lib.b200tfs_malloc(ctx, max(len(blob), 1), C.byref(arena)))
    a = np.frombuffer(blob, np.uint8)
    N.check(lib.b200tfs_memcpy_h2d(ctx, arena.value, a.ctypes.data, a.nbytes))
    n = len(wires)
    return arena.value, (C.c_uint64 * n)(*offs.tolist()), (C.c_uint64 * n)(*[len(w) for w in wires])


def graphed(lib, ctx, fn):
    N.check(lib.b200tfs_capture_begin(ctx))
    fn()
    g = C.c_void_p()
    N.check(lib.b200tfs_capture_end(ctx, C.byref(g)))
    return (lambda: N.check(lib.b200tfs_graph_launch(ctx, g))), g


def decode_legs(lib, ctx, timer, kinds, wires, calls, runs):
    n, T = len(wires), len(kinds)
    arena, off, ln = stage(lib, ctx, wires)
    cap = sum(int(x) // 2 for x in ln)
    dst = []
    for _ in range(2 * T):
        p = C.c_void_p()
        N.check(lib.b200tfs_malloc(ctx, 8 * cap, C.byref(p)))
        dst.append(p.value)
    kv = (C.c_int32 * T)(*kinds)
    vptr, lptr = (C.c_void_p * T)(*dst[:T]), (C.c_void_p * T)(*[dst[T + t] if k == M.CLASSIFY else None for t, k in enumerate(kinds)])
    caps, lcaps = (C.c_uint64 * T)(*[cap] * T), (C.c_uint64 * T)(*[cap if k == M.CLASSIFY else 0 for k in kinds])
    ref = M.expected(kinds, wires)

    def multi():
        N.check(lib.b200tfs_decode_multi_inference_responses(ctx, T, kv, arena, n, off, ln, vptr, caps, lptr, lcaps))

    # the same results as T separate Classify / Regress responses (each response's result t, re-framed as field 1)
    from tensorflow_serving.apis.classification_pb2 import ClassificationResponse
    from tensorflow_serving.apis.inference_pb2 import MultiInferenceResponse
    from tensorflow_serving.apis.regression_pb2 import RegressionResponse
    msgs = [MultiInferenceResponse.FromString(w) for w in wires]
    sep = []
    for t, k in enumerate(kinds):
        ws = []
        for m in msgs:
            r = ClassificationResponse() if k == M.CLASSIFY else RegressionResponse()
            r.model_spec.CopyFrom(m.results[t].model_spec)
            r.result.CopyFrom(m.results[t].classification_result if k == M.CLASSIFY else m.results[t].regression_result)
            ws.append(r.SerializeToString())
        sep.append((k, stage(lib, ctx, ws)))

    def separate():
        for t, (k, (a, o, ll)) in enumerate(sep):
            N.check(lib.b200tfs_decode_example_responses(ctx, k, a, n, o, ll, dst[t], cap, dst[T + t] if k == M.CLASSIFY else None,
                                                         cap if k == M.CLASSIFY else 0))

    def verify_multi():
        per, batch = (C.c_int64 * (3 * n * T))(), (C.c_int64 * (5 * T))()
        N.check(lib.b200tfs_multi_inference_response_results(ctx, n, T, per, None, batch))
        for t in range(T):
            assert batch[5 * t + 3] == N.OK
            v = np.empty(ref[t][0].size, np.uint32)
            N.check(lib.b200tfs_memcpy_d2h(ctx, v.ctypes.data, dst[t], v.nbytes))
            assert np.array_equal(v, np.ascontiguousarray(ref[t][0], np.float32).view(np.uint32).ravel())

    def verify_separate():
        # the last task's decode is the context's most recent one
        k = kinds[-1]
        per, batch = (C.c_int64 * (3 * n))(), (C.c_int64 * 5)()
        N.check(lib.b200tfs_example_response_results(ctx, n, per, None, batch))
        assert batch[3] == N.OK
        v = np.empty(ref[-1][0].size, np.uint32)
        N.check(lib.b200tfs_memcpy_d2h(ctx, v.ctypes.data, dst[T - 1], v.nbytes))
        assert np.array_equal(v, np.ascontiguousarray(ref[-1][0], np.float32).view(np.uint32).ravel()), k

    res = {}
    for name, fn, verify in (("multi", multi, verify_multi), ("classify+regress", separate, verify_separate)):
        ctx = fresh()     # a context of its own per leg: a captured graph pins the scratch of its context
        timer.ctx = ctx
        res[name + " eager"] = timer.run(fn, calls, runs)
        verify()
        g_fn, g = graphed(lib, ctx, fn)
        res[name + " graph"] = timer.run(g_fn, calls, runs)
        verify()
        N.check(lib.b200tfs_graph_destroy(g))
    return res


def encode_legs(lib, ctx, timer, calls, runs):
    rng = np.random.default_rng(3)
    n_req, n_ex = 256, 64
    tasks = [("head_c", CLASSIFY_METHOD_NAME), ("head_r", REGRESS_METHOD_NAME)]
    cols = [(rng.standard_normal((n_ex, 16)).astype(np.float32), rng.integers(0, 1 << 40, (n_ex, 4))) for _ in range(n_req)]
    keep, reqs = [], []
    for f, i in cols:
        fp, ip = C.c_void_p(), C.c_void_p()
        for p, a in ((fp, f), (ip, i)):
            N.check(lib.b200tfs_malloc(ctx, a.nbytes, C.byref(p)))
            N.check(lib.b200tfs_memcpy_h2d(ctx, p.value, a.ctypes.data, a.nbytes))
        fa = (N.Feature * 2)(N.Feature(data=fp.value, src_dtype=1, flags=N.F_DEVICE_DATA, row_elems=16, key=b"f", key_len=1),
                             N.Feature(data=ip.value, src_dtype=9, flags=N.F_DEVICE_DATA, row_elems=4, key=b"i", key_len=1))
        keep.append(fa)
        reqs.append(N.ExampleRequest(model_name=b"model", model_name_len=5, has_version=1, order=N.ORDER_UPB, version=1,
                                     n_examples=n_ex, n_features=2, flags=0, features=fa))
    ra = (N.ExampleRequest * n_req)(*reqs)
    sigs = [s.encode() for s, _ in tasks]
    arr = (N.InferenceTask * 2)(*[N.InferenceTask(signature_name=s, signature_len=len(s), method=m)
                                  for s, m in zip(sigs, (N.RESP_CLASSIFY, N.RESP_REGRESS))])
    ta = (N.ExampleTasks * n_req)(*[N.ExampleTasks(tasks=C.addressof(arr), n_tasks=2)] * n_req)
    res = {}
    for name, tk in (("multi", ta), ("classify", None)):
        ctx = fresh()
        timer.ctx = ctx
        cap = C.c_uint64()
        N.check(lib.b200tfs_example_tasks_arena_size(n_req, ra, None, None, None, None, tk, C.byref(cap)))
        p = C.c_void_p()
        N.check(lib.b200tfs_malloc(ctx, cap.value + 256, C.byref(p)))
        arena = (p.value + 255) & ~255

        def fn(tk=tk, arena=arena, cap=cap.value):
            N.check(lib.b200tfs_encode_example_tasks_async(ctx, n_req, ra, None, None, None, None, None, tk, arena, cap))

        def verify(arena=arena, tk=tk):
            off, ln = (C.c_uint64 * n_req)(), (C.c_uint64 * n_req)()
            N.check(lib.b200tfs_encode_results(ctx, n_req, off, ln))
            for r in (0, n_req // 2, n_req - 1):
                w = np.empty(ln[r], np.uint8)
                N.check(lib.b200tfs_memcpy_d2h(ctx, w.ctypes.data, arena + off[r], w.nbytes))
                d = {"f": cols[r][0], "i": cols[r][1]}
                if tk is None:
                    from min_tfs_client.requests import TensorServingClient
                    from tensorflow_serving.apis.classification_pb2 import ClassificationRequest
                    want = TensorServingClient._make_example_request(None, ClassificationRequest, "model", d, 1)
                else:
                    want = make_multi_inference_request("model", 1, tasks, d)
                assert w.tobytes() == want.SerializeToString(deterministic=True), r

        res[name + " eager"] = timer.run(fn, calls, runs)
        verify()
        g_fn, g = graphed(lib, ctx, fn)
        res[name + " graph"] = timer.run(g_fn, calls, runs)
        verify()
        N.check(lib.b200tfs_graph_destroy(g))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--json", metavar="PATH")
    args = ap.parse_args()
    lib = N.load()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print("GPU:", gpu)
    codec = get_codec()
    ctx = codec.ctx
    timer = Timer(lib, ctx)
    rng = np.random.default_rng(1)
    out = {"gpu": gpu}
    work = {"MI1": ([M.CLASSIFY, M.REGRESS], 256, 64), "MI2": ([M.CLASSIFY, M.REGRESS, M.CLASSIFY], 64, 1000)}
    for name, (kinds, n, rows) in work.items():
        wires = [M.random_response(rng, kinds, rows) for _ in range(n)]
        out[name] = decode_legs(lib, ctx, timer, kinds, wires, args.calls, args.runs)
    out["E2"] = encode_legs(lib, ctx, timer, args.calls, args.runs)
    for w in ("MI1", "MI2", "E2"):
        for leg, ts in out[w].items():
            print(f"{w:4s} {leg:26s} min {min(ts):9.1f} us   median {sorted(ts)[len(ts) // 2]:9.1f} us")
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
