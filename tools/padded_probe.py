"""Decode of a batch of PredictResponses with ragged trailing dims into one padded tensor per key (b200tfs_decode_padded), on three
workloads:

  P1  256 x {logits f32[1, T_r, 1024]}, T_r uniform in 32..512
  P2  1024 x {tokens int64[1, T_r] in 0..50 000, scores f32[1, T_r]}, T_r in 1..128
  P3  P1's shape at equal T (T = 272) - padded against b200tfs_decode_concat: what padding costs over concatenation

and three with DT_STRING outputs, decoded into padded offset-indexed byte columns (b200tfs_decode_padded_strings, pad b"[PAD]"):

  PS1  256 x {tokens string[1, T_r] of 1-16 B, logits f32[1, T_r, 32]}, T_r in 1..512   (detokenized tokens)
  PS2  1024 x {tags string[T_r, 5] of 3-10 B}, T_r in 1..64                              (NER tags, top-5 per token)
  PS3  64 x {text string[T_r] of 200-2000 B}, T_r in 1..16                               (long texts)

Legs (CUDA events around N calls after a warm-up, three runs each; the Python leg by the host clock):
  padded eager     b200tfs_decode_padded over a device arena
  padded graph     the same call captured once and replayed
  concat eager     b200tfs_decode_concat (P3 only)
  python           Codec.decode_predict_responses per response + numpy pad, host wire to host arrays
String legs: strings eager / strings graph (exact capacities from b200tfs_padded_strings_layout), today's
Codec.decode_predict_responses_padded (numpy str arrays decoded on the host; its ValueError is recorded where it raises),
string_columns=True end to end (host wire to host columns), and protobuf FromString plus numpy padding on one core.
Every leg is compared bit for bit against the numpy definition after its timed region.  The card's name and power limit are
read and printed by the same command.

    python tools/padded_probe.py [--iters 20] [--workloads P1,P2,P3,PS1,PS2,PS3]
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

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from concat_probe import _response, _string_tensor, _words  # noqa: E402


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


PAD = b"[PAD]"


def string_workload(name):
    rng = np.random.default_rng(0)
    if name == "PS1":
        return [_response([("tokens", _string_tensor(_words(rng, int(t), 1, 16), [1, int(t)])),
                           ("logits", O.encode_tensor_proto(rng.standard_normal((1, int(t), 32), dtype=np.float32)))])
                for t in rng.integers(1, 513, 256)], ["tokens", "logits"]
    if name == "PS2":
        return [_response([("tags", _string_tensor(_words(rng, 5 * int(t), 3, 10), [int(t), 5]))]) for t in rng.integers(1, 65, 1024)], ["tags"]
    return [_response([("text", _string_tensor(_words(rng, int(t), 200, 2000), [int(t)]))]) for t in rng.integers(1, 17, 64)], ["text"]


def padded_strings(wires, key):
    """The definition on one core: protobuf FromString, then the strings padded with PAD in numpy.  (offsets, data)."""
    from tensorflow_serving.apis import predict_pb2

    parts = []
    for w in wires:
        t = predict_pb2.PredictResponse.FromString(w).outputs[key]
        own = np.empty(len(t.string_val), object)
        own[:] = list(t.string_val)
        parts.append(own.reshape([int(d.size) for d in t.tensor_shape.dim]))
    tail = tuple(max(p.shape[d] for p in parts) for d in range(1, parts[0].ndim))
    res = np.empty((sum(p.shape[0] for p in parts), *tail), object)
    res.fill(PAD)
    r0 = 0
    for p in parts:
        res[(slice(r0, r0 + p.shape[0]),) + tuple(slice(0, d) for d in p.shape[1:])] = p
        r0 += p.shape[0]
    strs = res.ravel().tolist()
    offsets = np.zeros(len(strs) + 1, np.int64)
    np.cumsum(np.fromiter(map(len, strs), np.int64, len(strs)), out=offsets[1:])
    return offsets, np.frombuffer(b"".join(strs), np.uint8)


def run_strings(name, iters):
    wires, keys = string_workload(name)
    n, nk = len(wires), len(keys)
    codec = Codec(0)
    lib, ctx = codec._lib, codec.ctx
    buf, off, ln = codec._pack_wires(wires)
    arena = codec.device_array(buf)
    pk, ps = (N.PadKey * nk)(), (N.PaddedStrings * nk)()
    kb = [k.encode() for k in keys]
    for i, k in enumerate(kb):
        pk[i].key, pk[i].key_len = k, len(k)
    N.check(lib.b200tfs_padded_strings_layout(buf.ctypes.data, n, off, ln, nk, pk, ps, 0))
    skey = keys[0]
    want = padded_strings(wires, skey)
    bufs = []
    for i in range(nk):
        m = int(pk[i].bytes) // 8 - 1
        sizes = [("dst", int(pk[i].bytes))] + ([("data", int(ps[i].data_bytes) + (m - int(ps[i].strings)) * len(PAD))] if i == 0 else [])
        for attr, size in sizes:
            p = C.c_void_p()
            N.check(lib.b200tfs_malloc(ctx, max(size, 16), C.byref(p)))
            bufs.append((p, size))
            if attr == "dst":
                pk[i].dst, pk[i].dst_cap = p.value, size
            else:
                ps[i].data, ps[i].data_cap = p.value, size
    ps[0].pad, ps[0].pad_len = C.cast(C.c_char_p(PAD), C.c_void_p), len(PAD)

    def check(c, what):
        outs, st = (N.Output * (n * nk))(), (C.c_int32 * n)()
        N.check(c._lib.b200tfs_padded_results(c.ctx, n, nk, outs, None, st))
        assert all(outs[j].status == N.OK for j in range(n * nk)), f"{what}: the batch did not take the device route"
        o = np.empty(len(want[0]), np.int64)
        d = np.empty(len(want[1]), np.uint8)
        N.check(lib.b200tfs_memcpy_d2h(ctx, o.ctypes.data, pk[0].dst, o.nbytes))
        N.check(lib.b200tfs_memcpy_d2h(ctx, d.ctypes.data, ps[0].data, d.nbytes))
        codec.sync()
        assert o.tolist() == want[0].tolist() and d.tobytes() == want[1].tobytes(), what

    eager = lambda: N.check(lib.b200tfs_decode_padded_strings(ctx, arena.ptr, n, off, ln, nk, pk, ps))  # noqa: E731
    for _ in range(3):
        eager()
    t_eager = timed(codec, eager, iters)
    check(codec, "eager")
    gcodec = Codec(0)
    glib, gctx = gcodec._lib, gcodec.ctx
    gcall = lambda: N.check(glib.b200tfs_decode_padded_strings(gctx, arena.ptr, n, off, ln, nk, pk, ps))  # noqa: E731
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
        N.check(lib.b200tfs_memset(ctx, p.value, 0, max(size, 16)))
    codec.sync()
    N.check(glib.b200tfs_graph_launch(gctx, g))
    check(gcodec, "graph")
    N.check(glib.b200tfs_graph_destroy(g))

    def host_leg(fn, reps=3):
        ts, res = [], None
        for _ in range(reps):
            t0 = time.perf_counter()
            res = fn()
            ts.append(1e6 * (time.perf_counter() - t0))
        return ts, res
    try:
        t_today, today = host_leg(lambda: codec.decode_predict_responses_padded(wires, keys)[0])
        strs = [x.encode() for x in today[skey].ravel().tolist()]
        if strs != [want[1][a:b].tobytes() for a, b in zip(want[0][:-1], want[0][1:])]:
            t_today = ["differs from the definition (pads hold '0')"]
    except ValueError as e:   # numpy str arrays of different widths
        t_today = [f"raises ValueError ({str(e)[:60]}...)"]
    t_new, new = host_leg(lambda: codec.decode_predict_responses_padded(wires, keys, string_columns=True, string_pad=PAD)[0])
    assert new[skey].offsets.tolist() == want[0].tolist() and new[skey].data.tobytes() == want[1].tobytes(), "string_columns"
    t_pb, got = host_leg(lambda: padded_strings(wires, skey))
    assert got[0].tolist() == want[0].tolist() and got[1].tobytes() == want[1].tobytes(), "protobuf"
    for p, _ in bufs:
        lib.b200tfs_free(ctx, p)
    gcodec.close()
    codec.close()
    fmt = lambda xs: " / ".join(x if isinstance(x, str) else f"{x:.1f}" for x in xs)  # noqa: E731
    print(f"{name}: {n} records, {int(ps[0].strings)} strings in {len(want[0]) - 1} positions, "
          f"{len(want[1]) / 2**20:.2f} MiB of column bytes, {len(buf) / 2**20:.2f} MiB of wire")
    print(f"  strings eager      us/call {fmt(t_eager)}")
    print(f"  strings graph      us/call {fmt(t_graph)}")
    print(f"  today's padded     us {fmt(t_today)}   (numpy str, decoded on the host)")
    print(f"  string_columns     us {fmt(t_new)}   (decode_predict_responses_padded end to end, host wire to host columns)")
    print(f"  protobuf + numpy   us {fmt(t_pb)}   (FromString and numpy padding, one core)")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--workloads", default="P1,P2,P3,PS1,PS2,PS3")
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                          text=True).stdout.strip()
    print(f"card: {card}")
    for name in a.workloads.split(","):
        if name.startswith("PS"):
            run_strings(name, a.iters)
            continue
        res, wire, out = run(name, a.iters)
        print(f"{name}: wire {wire / 2**20:.1f} MiB, result {out / 2**20:.1f} MiB")
        for leg, us in res.items():
            print(f"  {leg:14s} " + " ".join(f"{u:10.1f}" for u in us) + " us/call")


if __name__ == "__main__":
    main()
