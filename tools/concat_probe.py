"""Decode of a batch of PredictResponses into one tensor per key (b200tfs_decode_concat) against the slot decode and the
Python route, on three workloads:

  A  256 x {scores f32[32,1000]}
  B  256 x {classes int64[32,5] (0..999), scores f32[32,5]}
  C  256 x {x f32[1024,1024]}  (a 1 GiB result)

and three with DT_STRING outputs, decoded into offset-indexed byte columns (b200tfs_decode_concat_strings):

  S1  256 x {classes string[32,5] of 1-12 B, scores f32[32,5]}   (a Predict-signature classifier)
  S2  256 x {text string[4] of 200-2000 B}                       (in-graph detokenisation)
  S3  64 x {labels string[64,1000] of 3-10 B}                    (many short strings per record)

Legs (CUDA events around N calls after a warm-up, three runs each; the Python leg by the host clock):
  concat eager     b200tfs_decode_concat over a device arena
  concat graph     the same call captured once and replayed
  slot decode      b200tfs_decode_responses of the same batch (record i into slot i)
  python           Codec.decode_predict_responses + np.concatenate, host wire to host arrays

String legs: strings eager / strings graph (as above, exact capacities from b200tfs_concat_strings_layout), today's
decode_predict_responses_concat (numpy str arrays, decoded on the host), the new Python call end to end (host wire to host
columns), and protobuf FromString plus a list of the strings on one core.  Every leg's bytes are compared after its timed region.
--profile adds a per-kernel split of the eager call from torch.profiler.

    python tools/concat_probe.py [--iters 20] [--workloads ABC] [--profile]
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


def _vi(x):
    out = bytearray()
    while True:
        out.append((x & 0x7F) | (0x80 if x > 0x7F else 0))
        x >>= 7
        if not x:
            return bytes(out)


def _ld(tag, b):
    return bytes([tag]) + _vi(len(b)) + b


def _string_tensor(strs, dims):
    shape = b"".join(_ld(0x12, b"\x08" + _vi(d) if d else b"") for d in dims)
    return b"\x08\x07" + _ld(0x12, shape) + b"".join(_ld(0x42, x) for x in strs)


def _response(entries):
    """A PredictResponse of (key, TensorProto bytes) entries and a model_spec."""
    spec = _ld(0x12, _ld(0x0A, b"default") + _ld(0x12, b"\x08\x01") + _ld(0x1A, b"serving_default"))
    return b"".join(_ld(0x0A, _ld(0x0A, k.encode()) + _ld(0x12, tp)) for k, tp in entries) + spec


def _words(rng, n, lo, hi):
    """n lower-case ASCII strings of lo..hi bytes (today's route converts to numpy str, which takes ASCII only)."""
    lens = rng.integers(lo, hi + 1, n)
    letters = rng.integers(97, 123, int(lens.sum()), dtype=np.uint8).tobytes()
    ends = np.cumsum(lens)
    return [letters[e - k: e] for e, k in zip(ends.tolist(), lens.tolist())]


def string_workload(name):
    rng = np.random.default_rng(0)
    if name == "S1":
        return [_response([("classes", _string_tensor(_words(rng, 160, 1, 12), [32, 5])),
                           ("scores", O.encode_tensor_proto(rng.standard_normal((32, 5), dtype=np.float32)))]) for _ in range(256)], ["classes", "scores"]
    if name == "S2":
        return [_response([("text", _string_tensor(_words(rng, 4, 200, 2000), [4]))]) for _ in range(256)], ["text"]
    return [_response([("labels", _string_tensor(_words(rng, 64000, 3, 10), [64, 1000]))]) for _ in range(64)], ["labels"]


def _reference_strings(wires, key):
    from tensorflow_serving.apis import predict_pb2

    return [x for w in wires for x in predict_pb2.PredictResponse.FromString(w).outputs[key].string_val]


def run_strings(name, iters, profile):
    wires, keys = string_workload(name)
    n, nk = len(wires), len(keys)
    codec = Codec(0)
    lib, ctx = codec._lib, codec.ctx
    buf, off, ln = codec._pack_wires(wires)
    arena = codec.device_array(buf)
    ck, sc = (N.ConcatKey * nk)(), (N.ConcatStrings * nk)()
    kb = [k.encode() for k in keys]
    for i, k in enumerate(kb):
        ck[i].key, ck[i].key_len = k, len(k)
    N.check(lib.b200tfs_concat_strings_layout(buf.ctypes.data, n, off, ln, nk, ck, sc, 0))
    bufs = []
    for i in range(nk):
        for attr, size in (("dst", int(ck[i].bytes)), ("data", int(sc[i].data_bytes))):
            p = C.c_void_p()
            N.check(lib.b200tfs_malloc(ctx, max(size, 1), C.byref(p)))
            bufs.append((p, size))
            if attr == "dst":
                ck[i].dst, ck[i].dst_cap = p.value, size
            else:
                sc[i].data, sc[i].data_cap = p.value, size
    strings = sum(int(sc[i].strings) for i in range(nk))
    data_bytes = sum(int(sc[i].data_bytes) for i in range(nk))
    ref = {k: _reference_strings(wires, k) for k in keys if int(ck[keys.index(k)].dtype) == 7}

    def check(c, what):
        outs, st = (N.Output * (n * nk))(), (C.c_int32 * n)()
        N.check(c._lib.b200tfs_concat_results(c.ctx, n, nk, outs, None, st))
        assert all(outs[j].status == N.OK for j in range(n * nk)), f"{what}: the batch did not take the device route"
        for i, k in enumerate(keys):
            if k not in ref:
                continue
            o = np.empty(int(ck[i].bytes) // 8, np.int64)
            d = np.empty(int(sc[i].data_bytes), np.uint8)
            N.check(lib.b200tfs_memcpy_d2h(ctx, o.ctypes.data, ck[i].dst, o.nbytes))
            N.check(lib.b200tfs_memcpy_d2h(ctx, d.ctypes.data, sc[i].data, d.nbytes))
            codec.sync()
            want = ref[k]
            assert o[0] == 0 and len(o) == len(want) + 1 and d.tobytes() == b"".join(want), (what, k)
            assert np.diff(o).tolist() == [len(x) for x in want], (what, k)

    eager = lambda: N.check(lib.b200tfs_decode_concat_strings(ctx, arena.ptr, n, off, ln, nk, ck, sc))  # noqa: E731
    for _ in range(3):
        eager()
    t_eager = timed(codec, eager, iters)
    check(codec, "eager")
    gcodec = Codec(0)
    glib, gctx = gcodec._lib, gcodec.ctx
    gcall = lambda: N.check(glib.b200tfs_decode_concat_strings(gctx, arena.ptr, n, off, ln, nk, ck, sc))  # noqa: E731
    gcall()
    gcodec.sync()
    N.check(glib.b200tfs_capture_begin(gctx))
    gcall()
    g = C.c_void_p()
    N.check(glib.b200tfs_capture_end(gctx, C.byref(g)))
    for _ in range(3):
        N.check(glib.b200tfs_graph_launch(gctx, g))
    t_graph = timed(gcodec, lambda: N.check(glib.b200tfs_graph_launch(gctx, g)), iters)
    for p, size in bufs:      # the graph wrote the same destinations: clear them, replay once more, check
        N.check(lib.b200tfs_memset(ctx, p.value, 0, max(size, 1)))
    codec.sync()
    N.check(glib.b200tfs_graph_launch(gctx, g))
    check(gcodec, "graph")
    N.check(glib.b200tfs_graph_destroy(g))

    def host_leg(fn, reps):
        ts, res = [], None
        for _ in range(reps):
            t0 = time.perf_counter()
            res = fn()
            ts.append(1e6 * (time.perf_counter() - t0))
        return ts, res
    reps = 3 if name != "S3" else 1
    try:
        t_today, today = host_leg(lambda: codec.decode_predict_responses_concat(wires, keys)[0], reps)
        for k in ref:
            assert [x.encode() for x in today[k].ravel().tolist()] == ref[k], ("today", k)
    except ValueError as e:   # numpy str arrays of different widths do not concatenate
        t_today = [f"raises ValueError ({str(e)[:60]}...)"]
    t_new, new = host_leg(lambda: codec.decode_predict_responses_concat(wires, keys, string_columns=True)[0], 3)
    for k in ref:
        o, d = new[k].offsets, new[k].data
        assert d.tobytes() == b"".join(ref[k]) and np.diff(o).tolist() == [len(x) for x in ref[k]], ("string_columns", k)

    def pb():
        from tensorflow_serving.apis import predict_pb2

        return [list(predict_pb2.PredictResponse.FromString(w).outputs[k].string_val) for w in wires for k in ref]
    t_pb, lists = host_leg(pb, reps)
    assert [x for lst in lists[: len(ref) * n: len(ref)] for x in lst] == ref[next(iter(ref))], "protobuf"
    split = _kernel_split(eager, codec) if profile else None
    for p, _ in bufs:
        lib.b200tfs_free(ctx, p)
    gcodec.close()
    codec.close()
    fmt = lambda xs: " / ".join(x if isinstance(x, str) else f"{x:.1f}" for x in xs)  # noqa: E731
    print(f"{name}: {n} records, {strings} strings, {data_bytes / 2**20:.2f} MiB of string bytes, {len(buf) / 2**20:.2f} MiB of wire")
    print(f"  strings eager      us/call {fmt(t_eager)}")
    print(f"  strings graph      us/call {fmt(t_graph)}")
    print(f"  today's concat     us {fmt(t_today)}   (numpy str, decoded on the host)")
    print(f"  string_columns     us {fmt(t_new)}   (decode_predict_responses_concat end to end, host wire to host columns)")
    print(f"  protobuf + list    us {fmt(t_pb)}   (FromString and list(string_val), one core)")
    if split:
        print("  per kernel (torch.profiler, us per call):")
        for k, us in split:
            print(f"    {us:9.1f}  {k}")


def _kernel_split(fn, codec, calls=10):
    """Device time per kernel name of `calls` calls of fn, from torch.profiler's CUDA activities."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        codec.sync()
    rows = []
    for e in prof.key_averages():
        dev = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
        if dev and "memcpy" not in e.key.lower():
            rows.append((e.key[:90], dev / calls))
    return sorted(rows, key=lambda r: -r[1])[:12]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--workloads", default="ABC", help="letters A B C, and / or S1 S2 S3 separated by commas (e.g. ABC,S1,S3)")
    ap.add_argument("--profile", action="store_true", help="a per-kernel split of the string workloads' eager call")
    args = ap.parse_args()
    try:
        print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv"], capture_output=True, text=True).stdout.strip())
    except OSError:
        print("nvidia-smi not found")
    for part in args.workloads.split(","):
        if part.startswith("S"):
            run_strings(part, args.iters, args.profile)
        else:
            for w in part:
                run(w, args.iters)


if __name__ == "__main__":
    main()
