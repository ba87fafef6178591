"""Classify / Regress request encode on the GPU (b200tfs_encode_example_requests_*) against the host path it replaces.

Workloads (one request each unless stated):
  W1  65 536 examples x {dense f32[64]}                                   float-only: closed-form offsets, no count / scan
  W2  16 384 examples x {dense f32[64], ids int64[8] in 0..50 000, age f32}
  W3  256 requests of 64 examples shaped like W2
  V1  16 384 examples x {history int64 ragged [16384, 64], lengths uniform in 0..64, values in 0..50 000; dense f32[64]}
  V2  65 536 examples x {emb f32 ragged [65536, 64], lengths uniform in 1..64}   float-only, but counted and scanned (beside W1)
  V3  4 096 examples x {tokens int32 ragged [4096, 512], lengths geometric with mean ~40, capped at 512}   worst-case emit spans
  V4  256 requests of 64 examples shaped like V1
  B1  65 536 examples x {country: 1 string of 2 B, tags: [n, 4] strings of 3-12 B, dense f32[16]}   bytes columns
  B2  16 384 examples x {query: 1 UTF-8 string of 100-400 B, ids int64[8] in 0..50 000}
  B3  256 requests of 64 examples shaped like B1
  W1P, W2P, V1P, B1P  W1, W2, V1 and B1 framed for Predict: a PredictRequest whose input "examples" is the DT_STRING [n] vector of the
      serialized examples (b200tfs_encode_example_targets_*), each run beside its Classify form
  K1  256 requests x 200 candidates {item f32[32], item_id int64} with a shared context {user f32[256], hist int64[50] in
      0..50 000, query: 1 string of 35 B}: an ExampleListWithContext (b200tfs_encode_example_contexts_*)
  K1R the same requests with the user features repeated in every example instead (B200TFS_F_BROADCAST rows, example_list)
  K1P K1 in the Predict-ELWC form: a PredictRequest whose input "examples" is the DT_STRING [1] serialized ExampleListWithContext
  K2  4 096 requests x 8 candidates shaped like K1: the context dominates, and each is written by its request's frame warp
  Q1  256 requests x 32 SequenceExamples: context {user f32[64], ids int64[4]}, lists {item_ids int64 ragged T <= 50,
      item_feats f32[T, 16] ragged} (b200tfs_encode_example_sequences_*, PREDICT_SEQUENCE)
  Q2  64 requests x 16 queries x 100 documents (TF-Ranking's SequenceExample form): context {query_len int64, query string},
      lists {doc_f0..doc_f7 f32, doc_title: one string of 5-30 B per step}
  Q3  256 requests x 16 sequences of 200 steps x 8 float lists of 2 values: about 21 KB each, above the 16 KB emit image
      (not in the default set; --workloads Q1,Q2,Q3; protobuf is timed once, _host over three calls)
  K3  64 requests x 16 queries x 100 candidates shaped like K1 (TF-Ranking's ELWC serving input, one ELWC per query): context
      {user f32[256], hist int64[50], query string} per query (b200tfs_encode_example_lists_*, PREDICT_ELWCS)
  K3R K3 with a ragged context `query_tokens` int64 [Q, 16], lengths 1..16
  K4  one request of 1 024 queries x 8 candidates: per-query headers and contexts dominate
      (not in the default set; --workloads K3,K3R,K4; beside each, the same queries as single-query PREDICT_ELWC requests through
      Codec.encode_example_requests, what a client sends today; protobuf is timed once, the Python legs over three calls)
  K5  K3 with list sizes in device memory (b200tfs_encode_example_device_lists_*): 64 requests x 16 queries over a capacity of
      N = 3 200 candidate rows each, every query's candidates drawn from 0..200 (so the total changes too), 8 such size sets
      cycled call after call
  K5L one request of 1 024 queries over N = 16 384 rows, each query's candidates drawn from 0..16 (K4's shape)
      (not in the default set; --workloads K5,K5L.  Legs: _async eager with host sizes, the host planning every call's new
      sizes; _async eager with device sizes; the graph captured once and replayed with device sizes.  Before each device-sizes
      call a device-to-device copy puts the next size set in place, as the GPU stage that produces them would; it is inside
      the timed region.  Bytes of both device legs are checked against protobuf for every size set after the timed region.)
Legs: the _async entry point eager (device columns -> device arena), the same captured once as a CUDA graph and replayed,
_host from pinned columns (copies both ways included), and examples_from_input_dict + SerializeToString(deterministic=True)
on one host core.  CUDA events over >= 20 calls after warm-up, three runs each; bytes = column bytes read + wire bytes
written; the share is of the H100 SXM data sheet's 3.35 TB/s.  W1 is set beside the Predict encode (b200tfs_encode_requests_async)
of the same f32[65536, 64] as one tensor, and W2 is split by kernel with torch.profiler in a run of its own.  Every leg's
bytes are checked against the host path after its timed region.  Needs a GPU; --json PATH also writes every number there.
The V workloads (ragged columns, b200tfs_encode_example_requests_ragged_*) count the values their lengths use, not the padded
columns, and the lengths; their host path builds the request one example at a time from the unchanged dense code, as a user
without ragged columns would.  The P workloads' host path is the one a Predict user has today: examples_from_input_dict,
SerializeToString(deterministic=True) of every example, string_val.extend and the PredictRequest's SerializeToString.
The B workloads (BytesColumn columns, b200tfs_encode_example_columns_*) count the string bytes and offsets; their host path runs
examples_from_input_dict over the equivalent numpy str / bytes arrays, which BytesColumn.from_array turns into the columns.
The K workloads' host path is examples_with_context_from_input_dict (K1R: examples_from_input_dict) and SerializeToString; K1R
counts its repeated rows once, as the kernels read them.
--profile V1,V3 runs only the per-kernel split of the named workloads (profiler on).

  python tools/example_probe.py [--calls 20] [--runs 3] [--workloads W1,V1,...] [--profile V1,V3] [--json PATH]
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
from min_tfs_client.codec import BytesColumn, Codec, RaggedColumn, _example_columns  # noqa: E402
from min_tfs_client.requests import TensorServingClient, examples_from_input_dict, examples_with_context_from_input_dict  # noqa: E402
from tensorflow.core.framework import types_pb2  # noqa: E402
from tensorflow_serving.apis.classification_pb2 import ClassificationRequest  # noqa: E402
from tensorflow_serving.apis.predict_pb2 import PredictRequest  # noqa: E402

PEAK = 3.35e12


def workloads(rng):
    def w2(n):
        return {"dense": rng.standard_normal((n, 64)).astype(np.float32), "ids": rng.integers(0, 50_000, (n, 8)),
                "age": rng.standard_normal(n).astype(np.float32)}
    def v1(n):
        return {"history": RaggedColumn(rng.integers(0, 50_000, (n, 64)), rng.integers(0, 65, n)),
                "dense": rng.standard_normal((n, 64)).astype(np.float32)}
    def tags(n):
        cells = rng.integers(97, 123, (n, 4, 12), dtype=np.uint8)
        cells[np.arange(12) >= rng.integers(3, 13, (n, 4, 1))] = 0
        return cells.view("S12").reshape(n, 4)
    def b1(n):
        return {"country": np.array([b"us", b"de", b"fr", b"jp", b"br"])[rng.integers(0, 5, n)], "tags": tags(n),
                "dense": rng.standard_normal((n, 16)).astype(np.float32)}
    def k1(n, repeated=False):
        d = {"item": rng.standard_normal((n, 32)).astype(np.float32), "item_id": rng.integers(0, 1 << 40, n)}
        ctx = {"user": rng.standard_normal(256).astype(np.float32), "hist": rng.integers(0, 50_000, 50),
               "query": BytesColumn.from_array(np.array(bytes(rng.integers(97, 123, 35, dtype=np.uint8))))}
        if not repeated:
            return d, ctx
        # the rows every example repeats: broadcast views, which build() passes as B200TFS_F_BROADCAST rows
        d.update(user=np.broadcast_to(ctx["user"], (n, 256)), hist=np.broadcast_to(ctx["hist"], (n, 50)), query=ctx["query"])
        return d
    words = ["".join(rng.choice(list("abcdefghij klmnop\u00e9\u00fc"), int(rng.integers(100, 400)))) for _ in range(1000)]
    queries = np.array([w.encode("utf-8")[:400].decode("utf-8", "ignore") for w in words])
    return {"W1": lambda: [{"dense": rng.standard_normal((65536, 64)).astype(np.float32)}], "W2": lambda: [w2(16384)],
            "W3": lambda: [w2(64) for _ in range(256)],
            "V1": lambda: [v1(16384)],
            "V2": lambda: [{"emb": RaggedColumn(rng.standard_normal((65536, 64)).astype(np.float32), rng.integers(1, 65, 65536))}],
            "V3": lambda: [{"tokens": RaggedColumn(rng.integers(0, 32_000, (4096, 512), dtype=np.int32),
                                                   np.minimum(rng.geometric(1 / 40, 4096), 512))}],
            "V4": lambda: [v1(64) for _ in range(256)],
            "W1P": lambda: [{"dense": rng.standard_normal((65536, 64)).astype(np.float32)}], "W2P": lambda: [w2(16384)],
            "V1P": lambda: [v1(16384)],
            "B1": lambda: [b1(65536)], "B1P": lambda: [b1(65536)], "B3": lambda: [b1(64) for _ in range(256)],
            "B2": lambda: [{"query": queries[rng.integers(0, 1000, 16384)], "ids": rng.integers(0, 50_000, (16384, 8))}],
            "K1": lambda: [k1(200) for _ in range(256)], "K1R": lambda: [k1(200, True) for _ in range(256)],
            "K1P": lambda: [k1(200) for _ in range(256)], "K2": lambda: [k1(8) for _ in range(4096)]}


def columns(d):
    """the device route's columns of a workload: numpy str / bytes arrays as BytesColumn"""
    return {k: BytesColumn.from_array(v) if isinstance(v, np.ndarray) and v.dtype.kind in "US" else v for k, v in d.items()}


def host_ref(d, predict=False, ctx=None):
    """the host path: examples_from_input_dict + SerializeToString; with ragged columns one example at a time (each example the
    one examples_from_input_dict makes of that example's rows), merged in order.  predict: every example serialized into the
    string_val of a PredictRequest's DT_STRING input "examples" instead.  ctx: an ExampleListWithContext, the Classify input or
    the one string_val"""
    if ctx is not None:
        req = TensorServingClient._make_example_request(None, ClassificationRequest, "model", d, 1, ctx)
        examples = [req.input.example_list_with_context]
    elif predict and not any(isinstance(v, RaggedColumn) for v in d.values()):
        examples = examples_from_input_dict(d).example_list.examples
    elif not any(isinstance(v, RaggedColumn) for v in d.values()):
        req = TensorServingClient._make_example_request(None, ClassificationRequest, "model", d, 1)
    else:
        req = TensorServingClient._make_example_request(None, ClassificationRequest, "model", {}, 1)
        n = next(v.shape[0] for v in d.values() if isinstance(v, RaggedColumn))
        for i in range(n):
            one = {k: v.values[i:i + 1, :int(v.lengths[i])] if isinstance(v, RaggedColumn) else v if np.ndim(v) == 0 else v[i:i + 1]
                   for k, v in d.items()}
            req.input.example_list.examples.extend(examples_from_input_dict(one).example_list.examples)
        examples = req.input.example_list.examples
    if not predict:
        return req.SerializeToString(deterministic=True)
    pr = PredictRequest()
    pr.model_spec.name = "model"
    pr.model_spec.version.value = 1
    t = pr.inputs["examples"]
    t.dtype = types_pb2.DT_STRING
    t.tensor_shape.dim.add().size = len(examples)
    t.string_val.extend(e.SerializeToString(deterministic=True) for e in examples)
    return pr.SerializeToString(deterministic=True)


def arrays(d):
    """the host arrays a request reads, in column order: values, then the lengths of a ragged column"""
    for v in d.values():
        if isinstance(v, RaggedColumn):
            yield v.values
            yield v.lengths
        elif isinstance(v, BytesColumn):
            yield v.data
            yield v.offsets
        else:
            yield v


def used_bytes(d):
    """column bytes the encode needs: a ragged column's used values and its lengths, every other column whole"""
    b = 0
    for v in d.values():
        if isinstance(v, np.ndarray) and v.ndim and not v.strides[0]:     # a repeated row, read once
            b += v[0].nbytes
        elif isinstance(v, RaggedColumn):
            unit = int(np.prod(v.shape[2:], dtype=np.int64))
            b += int(v.lengths.sum()) * unit * v.values.itemsize + v.lengths.nbytes
        elif isinstance(v, BytesColumn):
            b += v.data_len + v.offsets.nbytes
        else:
            b += np.asarray(v).nbytes
    return b


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


def build(dicts, device_ptrs=None, context=False):
    """(requests, ragged entries or None when no column is ragged, bytes entries or None when no column is one, keep-alive);
    device_ptrs[r]: the arrays(d) of request r in HBM.  A column of repeated rows (a broadcast view) is a B200TFS_F_BROADCAST
    row.  context: the dicts are contexts; the requests' features and n_features make their b200tfs_example_context entries"""
    keep, structs, ragged, strs = [], [], [], []
    for r, d in enumerate(dicts):
        n, preps = _example_columns(d, context=context)
        feats = (N.Feature * max(len(preps), 1))(*[p[0] for p in preps])
        for f, v in zip(feats, d.values()):
            if isinstance(v, np.ndarray) and v.ndim and not v.strides[0]:
                f.flags |= N.F_BROADCAST
        rg = [p[3] or N.Ragged() for p in preps]
        bs = [p.bytes_entry or N.Bytes() for p in preps]
        if device_ptrs is not None:
            ptrs = iter(device_ptrs[r])
            for f, g, b in zip(feats, rg, bs):
                f.data = next(ptrs)
                f.flags |= N.F_DEVICE_DATA
                if b.offsets:
                    b.offsets = next(ptrs)
                    b.flags = N.F_DEVICE_DATA
                if g.lengths:
                    g.lengths = next(ptrs)
                    g.flags = N.F_DEVICE_DATA
        ragged += rg
        strs += bs
        structs.append(N.ExampleRequest(model_name=b"model", model_name_len=5, has_version=1, order=N.ORDER_UPB, version=1,
                                        n_examples=n, n_features=len(preps), flags=0, features=feats))
        keep.append((preps, feats))
    rga = (N.Ragged * len(ragged))(*ragged) if any(g.lengths for g in ragged) else None
    bsa = (N.Bytes * len(strs))(*strs) if any(b.offsets for b in strs) else None
    return (N.ExampleRequest * len(structs))(*structs), rga, bsa, keep


def profile_split(lib, g, eager, calls):
    """per-kernel device time of `calls` eager encodes, profiler on"""
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            eager()
        N.check(lib.b200tfs_sync(g.ctx))
    split = {}
    for e in prof.key_averages():
        if "ex_" in e.key:
            total = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
            split[e.key] = {"count": e.count, "avg_us": total / max(e.count, 1)}
    return split


def sequence_workloads(rng):
    """the SequenceExample workloads: (context_dict, feature_list_dict) per request, host arrays"""
    def strs(m, lo, hi):
        lens = rng.integers(lo, hi + 1, m)
        return BytesColumn(rng.integers(97, 123, int(lens.sum())).astype(np.uint8), np.concatenate([[0], np.cumsum(lens)]))

    def q1():
        n, T = 32, 50
        lens = rng.integers(1, T + 1, n)
        return ({"user": rng.standard_normal((n, 64)).astype(np.float32), "ids": rng.integers(0, 1 << 40, (n, 4))},
                {"item_ids": RaggedColumn(rng.integers(0, 1 << 40, (n, T)), lens),
                 "item_feats": RaggedColumn(rng.standard_normal((n, T, 16)).astype(np.float32), lens)})

    def q2():
        n, T = 16, 100
        fl = {f"doc_f{j}": rng.standard_normal((n, T)).astype(np.float32) for j in range(8)}
        c = strs(n * T, 5, 30)
        fl["doc_title"] = BytesColumn(c.data, c.offsets, (n, T, 1))
        return {"query_len": rng.integers(1, 20, n), "query": strs(n, 3, 20)}, fl

    def q3():
        n, T = 16, 200
        return {"u": rng.standard_normal((n, 8)).astype(np.float32)}, \
            {f"l{j}": rng.standard_normal((n, T, 2)).astype(np.float32) for j in range(8)}

    return {"Q1": lambda: [q1() for _ in range(256)], "Q2": lambda: [q2() for _ in range(64)], "Q3": lambda: [q3() for _ in range(256)]}


def sequence_workload(name, pairs, args, codec, out):
    """_async eager, graph replay, _host and protobuf on one core for one SequenceExample workload; bytes compared afterwards"""
    import torch

    from min_tfs_client.codec import _sequence_count
    from min_tfs_client.requests import make_predict_sequence_examples_request

    def dev(v):
        if isinstance(v, RaggedColumn):
            return RaggedColumn(dev(v.values), torch.from_numpy(np.asarray(v.lengths, np.int64)).cuda())
        if isinstance(v, BytesColumn):
            return BytesColumn(torch.from_numpy(v.data).cuda(), torch.from_numpy(v.offsets).cuda(), v.shape)
        return torch.from_numpy(np.ascontiguousarray(v)).cuda()

    lib = N.load()
    g = Ctx()
    keep, structs, ragged, strs, seqs = [], [], [], [], []
    for ctx, fl in pairs:
        dctx, dfl = {k: dev(v) for k, v in ctx.items()}, {k: dev(v) for k, v in fl.items()}
        keep += [dctx, dfl]
        n = _sequence_count(ctx, fl)
        _, cp = _example_columns(dctx)
        _, lp = _example_columns(dfl)
        rg = [p[3] or N.Ragged() for p in cp]
        for p, v in zip(lp, fl.values()):
            r = p[3] or N.Ragged()
            r.max_len, r.unit = v.shape[1], int(np.prod(v.shape[2:], dtype=np.int64))
            rg.append(r)
        preps = cp + lp
        feats = (N.Feature * len(preps))(*[p[0] for p in preps])
        keep += [preps, feats]
        ragged += rg
        strs += [p.bytes_entry or N.Bytes() for p in preps]
        structs.append(N.ExampleRequest(model_name=b"model", model_name_len=5, has_version=1, order=N.ORDER_UPB, version=1,
                                        n_examples=n, n_features=len(preps), flags=0, features=feats))
        seqs.append(N.ExampleSequence(present=1, n_context=len(cp)))
    m = len(structs)
    reqs = (N.ExampleRequest * m)(*structs)
    rga, bsa = (N.Ragged * len(ragged))(*ragged), (N.Bytes * len(strs))(*strs)
    tga = (N.ExampleTarget * m)(*[N.ExampleTarget(kind=N.EXAMPLES_PREDICT_SEQUENCE, key=b"sequences", key_len=9)] * m)
    sqa = (N.ExampleSequence * m)(*seqs)
    cap = C.c_uint64()
    N.check(lib.b200tfs_example_sequences_arena_size(m, reqs, rga, bsa, tga, None, None, None, sqa, C.byref(cap)))
    arena = (g.malloc(cap.value + 256) + 255) & ~255

    def eager():
        N.check(lib.b200tfs_encode_example_sequences_async(g.ctx, m, reqs, rga, bsa, tga, None, None, None, sqa, arena, cap.value))

    eager()
    N.check(lib.b200tfs_encode_results(g.ctx, m, None, None))
    N.check(lib.b200tfs_capture_begin(g.ctx))
    eager()
    gr = C.c_void_p()
    N.check(lib.b200tfs_capture_end(g.ctx, C.byref(gr)))
    res = {"requests": m, "sequences": sum(s.n_examples for s in structs), "arena_bytes": cap.value}
    res["async_us"] = min(g.timed(eager, args.calls) for _ in range(args.runs))
    res["graph_us"] = min(g.timed(lambda: N.check(lib.b200tfs_graph_launch(g.ctx, gr)), args.calls) for _ in range(args.runs))
    items = [("model", 1, c, f) for c, f in pairs]
    res["host_us"] = min(timed_host(lambda: codec.encode_sequence_example_requests(items, input_key="sequences"), 3)
                         for _ in range(args.runs))
    t0 = time.perf_counter()
    refs = [make_predict_sequence_examples_request("model", 1, c, f, "sequences").SerializeToString(deterministic=True) for c, f in pairs]
    res["protobuf_one_core_us"] = (time.perf_counter() - t0) * 1e6
    res["wire_bytes"] = sum(len(w) for w in refs)
    # after the timed region: the replayed graph's and the host route's bytes against protobuf
    off, ln = (C.c_uint64 * m)(), (C.c_uint64 * m)()
    N.check(lib.b200tfs_graph_launch(g.ctx, gr))
    N.check(lib.b200tfs_encode_results(g.ctx, m, off, ln))
    host = np.empty(cap.value, np.uint8)
    N.check(lib.b200tfs_memcpy_d2h(g.ctx, host.ctypes.data, arena, cap.value))
    assert all(host[off[r]: off[r] + ln[r]].tobytes() == refs[r] for r in range(m)), name
    assert codec.encode_sequence_example_requests(items, input_key="sequences") == refs, name
    sizes = [int(s) for s in ln]
    res["max_request_bytes"] = max(sizes)
    N.check(lib.b200tfs_graph_destroy(gr))
    if name in args.profile.split(","):
        res["kernels"] = profile_split(lib, g, eager, args.calls)
    out["workloads"][name] = res
    print(name, res, flush=True)


def elwcs_workloads(rng):
    """the PREDICT_ELWCS workloads: (context_dict, input_dict, list_sizes) per request, host arrays"""
    def k3(Q, m, ragged=False):
        n = Q * m
        inp = {"item": rng.standard_normal((n, 32)).astype(np.float32), "item_id": rng.integers(0, 1 << 40, n)}
        q = rng.integers(97, 123, Q * 35).astype(np.uint8)
        ctx = {"user": rng.standard_normal((Q, 256)).astype(np.float32), "hist": rng.integers(0, 50_000, (Q, 50)),
               "query": BytesColumn(q, np.arange(Q + 1) * 35)}
        if ragged:
            ctx["query_tokens"] = RaggedColumn(rng.integers(0, 30_000, (Q, 16)), rng.integers(1, 17, Q))
        return ctx, inp, np.full(Q, m, np.int64)

    return {"K3": lambda: [k3(16, 100) for _ in range(64)], "K3R": lambda: [k3(16, 100, True) for _ in range(64)],
            "K4": lambda: [k3(1024, 8)]}


def elwcs_workload(name, items, args, codec, out):
    """_async eager, graph replay, _host and protobuf on one core for one PREDICT_ELWCS workload, and the same queries as
    single-query requests through the Python route; bytes compared afterwards"""
    import torch

    from min_tfs_client.requests import make_predict_elwcs_request

    def dev(v):
        if isinstance(v, RaggedColumn):
            return RaggedColumn(dev(v.values), torch.from_numpy(np.asarray(v.lengths, np.int64)).cuda())
        if isinstance(v, BytesColumn):
            return BytesColumn(torch.from_numpy(v.data).cuda(), torch.from_numpy(v.offsets).cuda(), v.shape)
        return torch.from_numpy(np.ascontiguousarray(v)).cuda()

    lib = N.load()
    g = Ctx()
    keep, structs, ragged, strs, lists, lragged, lstrs = [], [], [], [], [], [], []
    for ctx, inp, sizes in items:
        dctx, dinp = {k: dev(v) for k, v in ctx.items()}, {k: dev(v) for k, v in inp.items()}
        _, preps = _example_columns(dinp)
        _, cpreps = _example_columns(dctx)
        feats = (N.Feature * len(preps))(*[p[0] for p in preps])
        cfeats = (N.Feature * len(cpreps))(*[p[0] for p in cpreps])
        keep += [dctx, dinp, preps, cpreps, feats, cfeats, sizes]
        structs.append(N.ExampleRequest(model_name=b"model", model_name_len=5, has_version=1, order=N.ORDER_UPB, version=1,
                                        n_examples=int(sizes.sum()), n_features=len(preps), flags=0, features=feats))
        lists.append(N.ExampleLists(list_sizes=sizes.ctypes.data, n_lists=len(sizes), context=cfeats, n_context=len(cpreps), present=1))
        ragged += [p[3] or N.Ragged() for p in preps]
        strs += [p.bytes_entry or N.Bytes() for p in preps]
        lragged += [p[3] or N.Ragged() for p in cpreps]
        lstrs += [p.bytes_entry or N.Bytes() for p in cpreps]
    m = len(structs)
    reqs, lsa = (N.ExampleRequest * m)(*structs), (N.ExampleLists * m)(*lists)
    rga, bsa = (N.Ragged * len(ragged))(*ragged), (N.Bytes * len(strs))(*strs)
    lrga, lbsa = (N.Ragged * len(lragged))(*lragged), (N.Bytes * len(lstrs))(*lstrs)
    tga = (N.ExampleTarget * m)(*[N.ExampleTarget(kind=N.EXAMPLES_PREDICT_ELWCS, key=b"elwcs", key_len=5)] * m)
    cap = C.c_uint64()
    N.check(lib.b200tfs_example_lists_arena_size(m, reqs, rga, bsa, tga, None, None, None, None, None, lsa, lrga, lbsa, C.byref(cap)))
    arena = (g.malloc(cap.value + 256) + 255) & ~255

    def eager():
        N.check(lib.b200tfs_encode_example_lists_async(g.ctx, m, reqs, rga, bsa, tga, None, None, None, None, None, lsa, lrga, lbsa,
                                                       arena, cap.value))

    eager()
    N.check(lib.b200tfs_encode_results(g.ctx, m, None, None))
    N.check(lib.b200tfs_capture_begin(g.ctx))
    eager()
    gr = C.c_void_p()
    N.check(lib.b200tfs_capture_end(g.ctx, C.byref(gr)))
    res = {"requests": m, "queries": sum(len(s) for _, _, s in items), "examples": sum(int(s.sum()) for _, _, s in items),
           "arena_bytes": cap.value}
    for _ in range(3):
        eager()
    res["async_us"] = min(g.timed(eager, args.calls) for _ in range(args.runs))
    res["graph_us"] = min(g.timed(lambda: N.check(lib.b200tfs_graph_launch(g.ctx, gr)), args.calls) for _ in range(args.runs))
    calls = [("model", 1, c, i, s) for c, i, s in items]
    res["host_us"] = min(timed_host(lambda: codec.encode_elwc_requests(calls, input_key="elwcs"), 3) for _ in range(args.runs))
    t0 = time.perf_counter()
    refs = [make_predict_elwcs_request("model", 1, c, i, s, "elwcs").SerializeToString(deterministic=True) for c, i, s in items]
    res["protobuf_one_core_us"] = (time.perf_counter() - t0) * 1e6
    res["wire_bytes"] = sum(len(w) for w in refs)
    # the same queries as single-query Predict-ELWC requests (a ragged context has no such form)
    if not any(isinstance(v, RaggedColumn) for c, _, _ in items for v in c.values()):
        single = []
        for c, inp, sizes in items:
            s0 = np.concatenate([[0], np.cumsum(sizes)])
            for q in range(len(sizes)):
                cq = {k: BytesColumn(v.data, v.offsets[q: q + 2] - 0, (1,)) if isinstance(v, BytesColumn) else v[q] for k, v in c.items()}
                single.append(("model", 1, {k: v[s0[q]: s0[q + 1]] for k, v in inp.items()}, cq))
        res["single_query_requests"] = len(single)
        res["single_query_host_us"] = min(timed_host(lambda: codec.encode_example_requests(single, predict_input="elwcs"), 3)
                                          for _ in range(args.runs))
    # after the timed region: the replayed graph's and the host route's bytes against protobuf
    off, ln = (C.c_uint64 * m)(), (C.c_uint64 * m)()
    N.check(lib.b200tfs_graph_launch(g.ctx, gr))
    N.check(lib.b200tfs_encode_results(g.ctx, m, off, ln))
    host = np.empty(cap.value, np.uint8)
    N.check(lib.b200tfs_memcpy_d2h(g.ctx, host.ctypes.data, arena, cap.value))
    assert all(host[off[r]: off[r] + ln[r]].tobytes() == refs[r] for r in range(m)), name
    assert codec.encode_elwc_requests(calls, input_key="elwcs") == refs, name
    N.check(lib.b200tfs_graph_destroy(gr))
    if name in args.profile.split(","):
        res["kernels"] = profile_split(lib, g, eager, args.calls)
    out["workloads"][name] = res
    print(name, res, flush=True)


def elwcs_device_workloads(rng):
    """the PREDICT_ELWCS workloads with device list sizes: (context_dict, input_dict over N rows, [size sets]) per request"""
    def k5(Q, m_max, sets=8):
        n = Q * m_max
        inp = {"item": rng.standard_normal((n, 32)).astype(np.float32), "item_id": rng.integers(0, 1 << 40, n)}
        q = rng.integers(97, 123, Q * 35).astype(np.uint8)
        ctx = {"user": rng.standard_normal((Q, 256)).astype(np.float32), "hist": rng.integers(0, 50_000, (Q, 50)),
               "query": BytesColumn(q, np.arange(Q + 1) * 35)}
        return ctx, inp, [rng.integers(0, m_max + 1, Q).astype(np.int64) for _ in range(sets)]

    return {"K5": lambda: [k5(16, 200) for _ in range(64)], "K5L": lambda: [k5(1024, 16)]}


def elwcs_device_workload(name, items, args, out):
    """_async eager with host sizes (re-planned every call), _async eager with device sizes and the graph replayed with device
    sizes, over size sets that change call after call; every size set's bytes compared with protobuf afterwards"""
    import torch

    from min_tfs_client.requests import make_predict_elwcs_request

    lib = N.load()
    g = Ctx()
    m, S = len(items), len(items[0][2])
    keep, structs, strs, lists, lstrs = [], [], [], [], []
    for ctx, inp, size_sets in items:
        dctx = {k: BytesColumn(torch.from_numpy(v.data).cuda(), torch.from_numpy(v.offsets).cuda(), v.shape) if isinstance(v, BytesColumn)
                else torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in ctx.items()}
        dinp = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in inp.items()}
        _, preps = _example_columns(dinp)
        _, cpreps = _example_columns(dctx)
        feats = (N.Feature * len(preps))(*[p[0] for p in preps])
        cfeats = (N.Feature * len(cpreps))(*[p[0] for p in cpreps])
        keep += [dctx, dinp, preps, cpreps, feats, cfeats]
        n = next(iter(inp.values())).shape[0]
        structs.append(N.ExampleRequest(model_name=b"model", model_name_len=5, has_version=1, order=N.ORDER_UPB, version=1,
                                        n_examples=n, n_features=len(preps), flags=0, features=feats))
        lists.append(N.ExampleLists(list_sizes=None, n_lists=len(size_sets[0]), context=cfeats, n_context=len(cpreps), present=1))
        strs += [p.bytes_entry or N.Bytes() for p in preps]
        lstrs += [p.bytes_entry or N.Bytes() for p in cpreps]
    reqs, lsa = (N.ExampleRequest * m)(*structs), (N.ExampleLists * m)(*lists)
    bsa, lbsa = (N.Bytes * len(strs))(*strs), (N.Bytes * len(lstrs))(*lstrs)
    tga = (N.ExampleTarget * m)(*[N.ExampleTarget(kind=N.EXAMPLES_PREDICT_ELWCS, key=b"elwcs", key_len=5)] * m)
    # every size set of every request in device memory, and the live sizes buffer the encode reads
    Q = [len(it[2][0]) for it in items]
    q0 = np.concatenate([[0], np.cumsum(Q)]).astype(np.int64)
    sets = np.stack([np.concatenate([it[2][k] for it in items]) for k in range(S)]).astype(np.int64)     # [S, sum Q]
    dsets, live = g.malloc(sets.nbytes), g.malloc(sets[0].nbytes)
    N.check(lib.b200tfs_memcpy_h2d(g.ctx, dsets, sets.ctypes.data, sets.nbytes))
    dla = (N.ExampleDeviceLists * m)(*[N.ExampleDeviceLists(sizes=live + 8 * int(q0[r])) for r in range(m)])
    cap = C.c_uint64()
    N.check(lib.b200tfs_example_device_lists_arena_size(m, reqs, None, bsa, tga, None, None, None, None, None, lsa, None, lbsa, dla,
                                                        C.byref(cap)))
    arena = (g.malloc(cap.value + 256) + 255) & ~255
    step = [0]

    def next_sizes():
        k = step[0] % S
        step[0] += 1
        N.check(lib.b200tfs_memcpy_d2d(g.ctx, live, dsets + k * sets[0].nbytes, sets[0].nbytes))
        return k

    def device_eager():
        next_sizes()
        N.check(lib.b200tfs_encode_example_device_lists_async(g.ctx, m, reqs, None, bsa, tga, None, None, None, None, None, lsa, None,
                                                              lbsa, dla, arena, cap.value))

    # host sizes: the same columns, n_examples the set's total, planned on the host every call
    hreqs, hlsa = (N.ExampleRequest * m)(*structs), (N.ExampleLists * m)(*lists)

    def host_eager():
        k = step[0] % S
        step[0] += 1
        for r in range(m):
            hreqs[r].n_examples = int(sets[k, q0[r]: q0[r + 1]].sum())
            hlsa[r].list_sizes = sets[k].ctypes.data + 8 * int(q0[r])
        N.check(lib.b200tfs_encode_example_lists_async(g.ctx, m, hreqs, None, bsa, tga, None, None, None, None, None, hlsa, None, lbsa,
                                                       arena, cap.value))

    device_eager()
    N.check(lib.b200tfs_encode_results(g.ctx, m, None, None))
    N.check(lib.b200tfs_capture_begin(g.ctx))
    N.check(lib.b200tfs_encode_example_device_lists_async(g.ctx, m, reqs, None, bsa, tga, None, None, None, None, None, lsa, None, lbsa,
                                                          dla, arena, cap.value))
    gr = C.c_void_p()
    N.check(lib.b200tfs_capture_end(g.ctx, C.byref(gr)))

    def replay():
        next_sizes()
        N.check(lib.b200tfs_graph_launch(g.ctx, gr))

    res = {"requests": m, "queries": int(q0[-1]), "capacity_rows": sum(int(r.n_examples) for r in structs), "size_sets": S,
           "examples_per_set": [int(x) for x in sets.sum(axis=1)], "arena_bytes": cap.value}
    for leg, fn in (("host_sizes_async_us", host_eager), ("device_sizes_async_us", device_eager), ("device_sizes_graph_us", replay)):
        for _ in range(S):
            fn()
        res[leg] = [g.timed(fn, max(args.calls, S)) for _ in range(args.runs)]
    # after the timed region: every size set through both device legs against protobuf
    off, ln = (C.c_uint64 * m)(), (C.c_uint64 * m)()
    host = np.empty(cap.value, np.uint8)
    for k in range(S):
        refs = []
        for r, (ctx, inp, _) in enumerate(items):
            sz = sets[k, q0[r]: q0[r + 1]]
            t = int(sz.sum())
            refs.append(make_predict_elwcs_request("model", 1, ctx, {kk: v[:t] for kk, v in inp.items()}, sz, "elwcs")
                        .SerializeToString(deterministic=True))
        for fn in (device_eager, replay):
            step[0] = k
            fn()
            N.check(lib.b200tfs_encode_results(g.ctx, m, off, ln))
            N.check(lib.b200tfs_memcpy_d2h(g.ctx, host.ctypes.data, arena, cap.value))
            N.check(lib.b200tfs_sync(g.ctx))
            assert all(host[off[r]: off[r] + ln[r]].tobytes() == refs[r] for r in range(m)), (name, k)
    res["bytes_checked_sets"] = S
    N.check(lib.b200tfs_graph_destroy(gr))
    out["workloads"][name] = res
    print(name, res, flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--workloads", default="W1,W1P,W2,W2P,W3,V1,V1P,V2,V3,V4,B1,B1P,B2,B3", help="comma-separated workloads to run")
    ap.add_argument("--profile", default="", help="only the per-kernel split of these workloads (comma-separated)")
    ap.add_argument("--json", metavar="PATH", help="write every number of the run to PATH as JSON")
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    rng = np.random.default_rng(0)
    W = workloads(rng)
    lib = N.load()
    codec = Codec(0)
    out = {"card": card, "calls": args.calls, "runs": args.runs, "workloads": {}}
    profile_only = [w for w in args.profile.split(",") if w]
    Q = sequence_workloads(rng)
    K = elwcs_workloads(rng)
    KD = elwcs_device_workloads(rng)
    for name in (profile_only or args.workloads.split(",")):
        if name in Q:
            sequence_workload(name, Q[name](), args, codec, out)
            continue
        if name in K:
            elwcs_workload(name, K[name](), args, codec, out)
            continue
        if name in KD:
            elwcs_device_workload(name, KD[name](), args, out)
            continue
        pairs = [x if isinstance(x, tuple) else (x, None) for x in W[name]()]
        host_dicts = [d for d, _ in pairs]
        host_ctxs = [c for _, c in pairs]
        with_ctx = host_ctxs[0] is not None
        dicts = [columns(d) for d in host_dicts]
        predict = name.endswith("P")
        g = Ctx()       # a context per workload: the graph captured below pins its scratch buffers
        refs = [host_ref(d, predict, c) for d, c in pairs]
        col_bytes = sum(used_bytes(d) for d in dicts) + (sum(used_bytes(c) for c in host_ctxs) if with_ctx else 0)
        wire_bytes = sum(len(w) for w in refs)
        moved = col_bytes + wire_bytes
        # device columns
        def upload(ds):
            ptrs = []
            for d in ds:
                row = []
                for a in arrays(d):
                    if isinstance(a, np.ndarray) and a.ndim and not a.strides[0]:
                        a = np.ascontiguousarray(a[0])          # a repeated row: its one row
                    p = g.malloc(a.nbytes)
                    N.check(lib.b200tfs_memcpy_h2d(g.ctx, p, a.ctypes.data, a.nbytes))
                    row.append(p)
                ptrs.append(row)
            return ptrs
        ptrs = upload(dicts)
        reqs, rga, bsa, keep = build(dicts, ptrs)
        n = len(dicts)
        kind = N.EXAMPLES_PREDICT_ELWC if with_ctx else N.EXAMPLES_PREDICT_STRING
        tg = (N.ExampleTarget * n)(*[N.ExampleTarget(kind=kind, key=b"examples", key_len=8)] * n) if predict else None
        def contexts(cdicts, cptrs=None):
            """(b200tfs_example_context entries, their bytes entries, keep-alive)"""
            creqs, _, cbsa, ckeep = build(cdicts, cptrs, context=True)
            ct = (N.ExampleContext * n)(*[N.ExampleContext(features=q.features, n_features=q.n_features, present=1) for q in creqs])
            return ct, cbsa, (creqs, ckeep)
        ct = cbsa = None
        if with_ctx:
            ct, cbsa, ckeep = contexts(host_ctxs, upload(host_ctxs))
        cap = C.c_uint64()
        N.check(lib.b200tfs_example_context_arena_size(n, reqs, bsa, tg, ct, cbsa, C.byref(cap)))
        arena = g.malloc(cap.value)
        off, ln = (C.c_uint64 * n)(), (C.c_uint64 * n)()

        def eager():
            if with_ctx:
                N.check(lib.b200tfs_encode_example_contexts_async(g.ctx, n, reqs, rga, bsa, tg, ct, cbsa, arena, cap.value))
            elif bsa is not None:
                N.check(lib.b200tfs_encode_example_columns_async(g.ctx, n, reqs, rga, bsa, tg, arena, cap.value))
            elif predict:
                N.check(lib.b200tfs_encode_example_targets_async(g.ctx, n, reqs, rga, tg, arena, cap.value))
            elif rga is None:
                N.check(lib.b200tfs_encode_example_requests_async(g.ctx, n, reqs, arena, cap.value))
            else:
                N.check(lib.b200tfs_encode_example_requests_ragged_async(g.ctx, n, reqs, rga, arena, cap.value))

        if profile_only:
            for _ in range(3):
                eager()
            N.check(lib.b200tfs_sync(g.ctx))
            split = profile_split(lib, g, eager, args.calls)
            out[f"{name}_kernels"] = split
            print(name, "kernels", json.dumps(split), flush=True)
            continue

        def check_arena():
            N.check(lib.b200tfs_encode_results(g.ctx, n, off, ln))
            for i in range(n):
                buf = np.empty(ln[i], np.uint8)
                N.check(lib.b200tfs_memcpy_d2h(g.ctx, buf.ctypes.data, arena + off[i], ln[i]))
                N.check(lib.b200tfs_sync(g.ctx))
                assert buf.tobytes() == refs[i], (name, i)

        res = {"column_bytes": col_bytes, "wire_bytes": wire_bytes, "wire_bytes_per_request": wire_bytes / n}
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
        def pin(a):
            p = codec.pinned_empty(np.shape(a), np.asarray(a).dtype)
            p[...] = a
            return p
        def pin_col(v):
            if isinstance(v, np.ndarray) and v.ndim and not v.strides[0]:
                return np.broadcast_to(pin(v[0]), v.shape)
            if isinstance(v, RaggedColumn):
                return RaggedColumn(pin(v.values), pin(v.lengths))
            if isinstance(v, BytesColumn):
                return BytesColumn(pin(v.data), pin(v.offsets), v.shape)
            return pin(v)
        pinned = [{k: pin_col(v) for k, v in d.items()} for d in dicts]
        hreqs, hrga, hbsa, hkeep = build(pinned)
        wire = N.PinnedBuffer(cap.value)
        hoff, hln = (C.c_uint64 * n)(), (C.c_uint64 * n)()
        if with_ctx:
            hct, hcbsa, hckeep = contexts([{k: pin_col(v) for k, v in c.items()} for c in host_ctxs])
            host = lambda: N.check(lib.b200tfs_encode_example_contexts_host(codec.ctx, n, hreqs, hrga, hbsa, tg, hct, hcbsa,  # noqa: E731
                                                                             wire.ptr, cap.value, hoff, hln))
        elif hbsa is not None:
            host = lambda: N.check(lib.b200tfs_encode_example_columns_host(codec.ctx, n, hreqs, hrga, hbsa, tg, wire.ptr, cap.value,  # noqa: E731
                                                                            hoff, hln))
        elif predict:
            host = lambda: N.check(lib.b200tfs_encode_example_targets_host(codec.ctx, n, hreqs, hrga, tg, wire.ptr, cap.value,  # noqa: E731
                                                                            hoff, hln))
        elif hrga is None:
            host = lambda: N.check(lib.b200tfs_encode_example_requests_host(codec.ctx, n, hreqs, wire.ptr, cap.value, hoff, hln))  # noqa: E731
        else:
            host = lambda: N.check(lib.b200tfs_encode_example_requests_ragged_host(codec.ctx, n, hreqs, hrga, wire.ptr, cap.value,  # noqa: E731
                                                                                    hoff, hln))
        for _ in range(3):
            host()
        res["host_pinned_us"] = [timed_host(host, args.calls) for _ in range(args.runs)]
        assert all(wire.array[hoff[i]: hoff[i] + hln[i]].tobytes() == refs[i] for i in range(n)), name
        # the host path it replaces, one core
        runs = []
        for _ in range(args.runs):
            t0 = time.perf_counter()
            for d, c in pairs:
                host_ref(d, predict, c)
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
        if name in ("W2", "B1", "B2", "K1", "K1R", "K2"):     # per-kernel split, profiler on, in a run of its own
            split = profile_split(lib, g, eager, args.calls)
            out[f"{name}_kernels"] = split
            print(name, "kernels", json.dumps(split), flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)
    codec.close()


if __name__ == "__main__":
    main()
