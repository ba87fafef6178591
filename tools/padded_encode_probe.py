"""Time Codec.encode_predict_requests_padded / b200tfs_encode_padded_requests_async against the status quo, and compare every leg's
bytes after its timed region.

Workloads (sequence and image clients whose batch is already on the GPU):
  U1  1024 x {input_ids, attention_mask: int64[1, T_r]} from int64[1024, 512], T_r in 16..512, ids in 0..50000
  U2  256 x f32[1, T_r, 1024] from f32[256, 512, 1024]
  U3  the split of f32[262144, 1024] into 256 x f32[1024, 1024]
  U4  64 x f32[1, H_r, W_r, 3] from f32[64, 512, 512, 3]
String workloads (DT_STRING inputs from a BytesColumn on the device; --strings runs these alone):
  T1  1024 x {text: string[rows_r], ids: int64[rows_r]}, rows_r in 1..64, strings of 16..256 bytes
  T2  256 x text: string[rows_r, S_r1] from string[R, 8], rows_r in 1..32, S_r1 in 1..8, strings of 16..64 bytes
  T3  64 x image_bytes: string[1], one binary string of 256 KiB - 2 MiB each
  legs: device (eager and graph, as above), today (a numpy str_ column through the host route; T3 has none: binary data cannot be
  a str_ array) and protobuf (the requests built and serialized with the protobuf runtime on one host core).
Legs:
  device  the C call, eager (host call to results, arena ready on the device) and as a replayed CUDA graph
  quo     the status quo: shapes to the host, a synchronise, per-request structs over the device boxes planned on the host, then
          b200tfs_encode_requests_async; the wire stays on the device, as in the device legs (contiguous boxes only: U1-U3)
  existing  the same b200tfs_encode_requests_async with the requests planned once: the existing encode at equal bytes
  python  Codec.encode_predict_requests_padded (bytes on the host)
  defn    the definition: host slicing, then encode_predict_requests
Usage: python tools/padded_encode_probe.py [--strings] [out.json]
GB/s = (source bytes read + wire bytes written) / time; share of the H100 SXM's 3.35 TB/s.
"""
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.join(HERE, "..", "min-tfs-client_b200"), os.path.join(HERE, ".."), os.path.join(HERE, "..", "tests")]

import torch  # noqa: E402

from min_tfs_client import _native as N  # noqa: E402
from min_tfs_client.codec import BytesColumn, Codec  # noqa: E402
import padded_strings_ref as SR  # noqa: E402


def workloads(rng):
    T = rng.integers(16, 513, 1024)
    ids = torch.from_numpy(rng.integers(0, 50001, (1024, 512))).cuda()
    yield "U1", {"input_ids": ids, "attention_mask": torch.ones_like(ids)}, np.stack([np.ones(1024, np.int64), T], 1), True
    T = rng.integers(16, 513, 256)
    yield "U2", {"x": torch.randn(256, 512, 1024, device="cuda")}, np.stack([np.ones(256, np.int64), T, np.full(256, 1024)], 1), True
    yield "U3", {"x": torch.randn(262144, 1024, device="cuda")}, np.full(256, 1024, np.int64), True
    H, W = rng.integers(64, 513, 64), rng.integers(64, 513, 64)
    yield "U4", {"image": torch.randn(64, 512, 512, 3, device="cuda")}, np.stack([np.ones(64, np.int64), H, W, np.full(64, 3)], 1), False


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(reps):
        out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) / reps, out


def string_workloads(rng):
    """(name, strings, dims, shapes, numeric padded inputs, text strings?) of T1-T3"""
    def text(m, lo, hi):
        lens = rng.integers(lo, hi + 1, m)
        letters = rng.integers(97, 123, int(lens.sum())).astype(np.uint8).tobytes()
        off = np.concatenate([[0], np.cumsum(lens)])
        return [letters[off[j]: off[j + 1]] for j in range(m)]
    rows = rng.integers(1, 65, 1024).astype(np.int64)
    R = int(rows.sum())
    yield "T1", text(R, 16, 256), (R,), rows, {"ids": rng.integers(0, 1 << 40, R)}, True
    rows = rng.integers(1, 33, 256).astype(np.int64)
    R = int(rows.sum())
    yield "T2", text(R * 8, 16, 64), (R, 8), np.stack([rows, rng.integers(1, 9, 256)], 1), {}, True
    sizes = rng.integers(256 << 10, (2 << 20) + 1, 64)
    yield "T3", [rng.integers(0, 256, int(k)).astype(np.uint8).tobytes() for k in sizes], (64,), np.ones(64, np.int64), {}, False


def run_strings(codec, lib, rng, out):
    for name, strs, dims, shapes, numeric, is_text in string_workloads(rng):
        n = len(shapes)
        key = "image_bytes" if name == "T3" else "text"
        lens = np.array([len(x) for x in strs], np.int64)
        offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        data_h = np.frombuffer(b"".join(strs), np.uint8)
        data, offsets = torch.from_numpy(data_h.copy()).cuda(), torch.from_numpy(offs).cuda()
        col = BytesColumn(data, offsets, dims)
        num = {k: torch.from_numpy(v).cuda() for k, v in numeric.items()}
        S = {key: torch.from_numpy(np.ascontiguousarray(shapes)).cuda(), **{k: torch.from_numpy(np.ascontiguousarray(shapes.reshape(n, -1)[:, 0])).cuda()
                                                                             for k in numeric}}
        ref = SR.reference_requests("m", 1, {key: (strs, dims), **numeric}, {k: s.cpu().numpy() for k, s in S.items()}, {})
        # source bytes: the strings of the boxes, their offsets and the numeric boxes; wire bytes: the requests
        box_bytes, box_strs, r0 = 0, 0, 0
        for r in range(n):
            row = shapes.reshape(n, -1)[r]
            bs, _ = SR.box_strings(list(range(len(strs))), dims, r0, row)
            box_bytes += int(lens[bs].sum())
            box_strs += len(bs)
            r0 += int(row[0])
        src = box_bytes + 16 * box_strs + sum(8 * int(shapes.reshape(n, -1)[:, 0].sum()) for _ in numeric)
        wire_bytes = sum(len(w) for w in ref)
        reps = 5
        res = {}
        # the C call, eager and as a replayed graph
        keep, structs, pins, bts = [], [], [], []
        for k, t in [(key, None)] + list(num.items()):
            if t is None:
                d = (C.c_int64 * len(dims))(*dims)
                structs.append(N.Tensor(data=data.data_ptr(), src_dtype=7, wire_dtype=7, rank=len(dims), flags=N.F_DEVICE_DATA, dims=d,
                                        key=k.encode(), key_len=len(k), packed_len=0))
                bts.append(N.Bytes(offsets=offsets.data_ptr(), data_len=data_h.size, flags=N.F_DEVICE_DATA))
            else:
                d = (C.c_int64 * 1)(t.shape[0])
                structs.append(N.Tensor(data=t.data_ptr(), src_dtype=9, wire_dtype=9, rank=1, flags=N.F_DEVICE_DATA, dims=d, key=k.encode(),
                                        key_len=len(k), packed_len=0))
                bts.append(N.Bytes())
            keep.append(d)
            pins.append(N.PadInput(shapes=S[k].data_ptr(), cols=S[k].shape[1] if S[k].dim() == 2 else 1))
        arr = (N.Tensor * len(structs))(*structs)
        req = N.Request(model_name=b"m", model_name_len=1, has_version=1, order=N.ORDER_UPB, version=1, n_inputs=len(structs), flags=0, inputs=arr)
        pin_arr, bt_arr = (N.PadInput * len(pins))(*pins), (N.Bytes * len(bts))(*bts)
        cap = C.c_uint64()
        N.check(lib.b200tfs_padded_request_columns_arena_size(n, C.byref(req), bt_arr, C.byref(cap)))
        gc = Codec(0)
        mem = C.c_void_p()
        N.check(lib.b200tfs_malloc(gc.ctx, cap.value, C.byref(mem)))
        arena = mem.value
        off, ln = (C.c_uint64 * n)(), (C.c_uint64 * n)()

        def wires():
            N.check(lib.b200tfs_encode_results(gc.ctx, n, off, ln))
            end = max(int(off[i]) + int(ln[i]) for i in range(n))
            host = np.empty(end, np.uint8)
            N.check(lib.b200tfs_memcpy_d2h(gc.ctx, host.ctypes.data, arena, end))
            gc.sync()
            return [host[off[i]: off[i] + ln[i]].tobytes() for i in range(n)]

        def eager():
            N.check(lib.b200tfs_encode_padded_requests_columns_async(gc.ctx, n, C.byref(req), pin_arr, bt_arr, arena, cap.value))
            gc.sync()

        res["device"], _ = timed(eager, reps)
        assert wires() == ref, f"{name}: device bytes differ"
        N.check(lib.b200tfs_capture_begin(gc.ctx))
        N.check(lib.b200tfs_encode_padded_requests_columns_async(gc.ctx, n, C.byref(req), pin_arr, bt_arr, arena, cap.value))
        g = C.c_void_p()
        N.check(lib.b200tfs_capture_end(gc.ctx, C.byref(g)))

        def replay():
            N.check(lib.b200tfs_graph_launch(gc.ctx, g.value))
            gc.sync()

        res["graph"], _ = timed(replay, reps)
        assert wires() == ref, f"{name}: graph replay bytes differ"
        N.check(lib.b200tfs_graph_destroy(g.value))
        N.check(lib.b200tfs_free(gc.ctx, arena))
        gc.close()
        dt, got = timed(lambda: codec.encode_predict_requests_padded("m", {key: col, **num}, S, model_version=1), reps)
        assert got == ref, f"{name}: python bytes differ"
        res["python"] = dt
        if is_text:     # today's route: a numpy str_ column, sliced and encoded request by request on the host
            a = np.array([x.decode() for x in strs]).reshape(dims)
            hs = {k: s.cpu().numpy() for k, s in S.items()}
            dt, got = timed(lambda: codec._padded_requests_on_host("m", 1, {key: a, **numeric}, hs, {}, n), 1)
            assert got == ref, f"{name}: today's bytes differ"
            res["today"] = dt
        hs = {k: s.cpu().numpy() for k, s in S.items()}
        dt, got = timed(lambda: SR.reference_requests("m", 1, {key: (strs, dims), **numeric}, hs, {}), 1)
        assert got == ref
        res["protobuf"] = dt
        line = {"workload": name, "n": n, "src_bytes": src, "wire_bytes": wire_bytes}
        for leg, t in res.items():
            gbs = (src + wire_bytes) / t / 1e9
            line[leg] = {"us": round(t * 1e6, 1), "GB/s": round(gbs, 2)}
        print(json.dumps(line))
        out["workloads"][name] = line
        del data, offsets, col, num, S
        torch.cuda.empty_cache()


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("card:", q)
    codec = Codec(0)
    lib = N.load()
    rng = np.random.default_rng(0)
    out = {"card": q, "workloads": {}}
    only_strings = "--strings" in sys.argv
    args = [a for a in sys.argv[1:] if a != "--strings"]
    run_strings(codec, lib, np.random.default_rng(1), out)
    for name, inputs, shapes, contiguous in ([] if only_strings else workloads(rng)):
        torch.cuda.synchronize()
        S = {k: torch.from_numpy(shapes[:, :t.dim()] if shapes.ndim == 2 else shapes).cuda().contiguous() for k, t in inputs.items()}
        src = 0
        for k, t in inputs.items():
            s = shapes.reshape(len(shapes), -1)
            per = np.prod(s[:, : t.dim()], axis=1) if s.shape[1] > 1 else s[:, 0] * int(np.prod(t.shape[1:]))
            src += int(per.sum()) * t.element_size()
        reps = 5
        res = {}
        # the Python call
        dt, wires = timed(lambda: codec.encode_predict_requests_padded("m", inputs, S, model_version=1), reps)
        wire_bytes = sum(len(w) for w in wires)
        res["python"] = dt
        # the C call over the codec's own arena, eager and as a graph (the arena the Python call sized)
        keep = []
        structs, pins = [], []
        for k, t in inputs.items():
            dims = (C.c_int64 * t.dim())(*t.shape)
            keep.append(dims)
            e = 1 if t.dtype == torch.float32 else 9
            structs.append(N.Tensor(data=t.data_ptr(), src_dtype=e, wire_dtype=e, rank=t.dim(), flags=N.F_DEVICE_DATA, dims=dims, key=k.encode(),
                                    key_len=len(k), packed_len=0))
            pins.append(N.PadInput(shapes=S[k].data_ptr(), cols=S[k].shape[1] if S[k].dim() == 2 else 1))
        arr = (N.Tensor * len(structs))(*structs)
        req = N.Request(model_name=b"m", model_name_len=1, has_version=1, order=N.ORDER_UPB, version=1, n_inputs=len(structs), flags=0, inputs=arr)
        pin_arr = (N.PadInput * len(pins))(*pins)
        cap = C.c_uint64()
        N.check(lib.b200tfs_padded_request_arena_size(len(shapes), C.byref(req), C.byref(cap)))
        n = len(shapes)
        gc = Codec(0)         # a context of its own: a captured graph pins its context's scratch buffers
        arena_mem = C.c_void_p()
        N.check(lib.b200tfs_malloc(gc.ctx, cap.value, C.byref(arena_mem)))
        arena = arena_mem.value

        def eager():
            N.check(lib.b200tfs_encode_padded_requests_async(gc.ctx, n, C.byref(req), pin_arr, arena, cap.value))
            gc.sync()

        res["device"], _ = timed(eager, reps)
        N.check(lib.b200tfs_capture_begin(gc.ctx))
        N.check(lib.b200tfs_encode_padded_requests_async(gc.ctx, n, C.byref(req), pin_arr, arena, cap.value))
        g = C.c_void_p()
        N.check(lib.b200tfs_capture_end(gc.ctx, C.byref(g)))

        def replay():
            N.check(lib.b200tfs_graph_launch(gc.ctx, g.value))
            gc.sync()

        res["graph"], _ = timed(replay, reps)
        off, ln = (C.c_uint64 * n)(), (C.c_uint64 * n)()
        N.check(lib.b200tfs_encode_results(gc.ctx, n, off, ln))
        end = max(int(off[i]) + int(ln[i]) for i in range(n))
        host = np.empty(end, np.uint8)
        N.check(lib.b200tfs_memcpy_d2h(gc.ctx, host.ctypes.data, arena, end))
        gc.sync()
        assert [host[off[i]: off[i] + ln[i]].tobytes() for i in range(n)] == wires, f"{name}: graph replay bytes differ"
        N.check(lib.b200tfs_graph_destroy(g.value))
        N.check(lib.b200tfs_free(gc.ctx, arena))
        gc.close()
        if contiguous:
            qc = Codec(0)

            def plan_quo(sh):
                # per-request structs over the device boxes (contiguous here), planned on the host
                keep_q, reqs_q = [], []
                r0 = {k: 0 for k in inputs}
                for r in range(n):
                    ts = []
                    for k, t in inputs.items():
                        row = [int(x) for x in sh[k][r]] + list(t.shape[len(sh[k][r]):])
                        dims = (C.c_int64 * len(row))(*row)
                        pitch = t.element_size() * int(np.prod(t.shape[1:]))
                        e = 1 if t.dtype == torch.float32 else 9
                        ts.append(N.Tensor(data=t.data_ptr() + r0[k] * pitch, src_dtype=e, wire_dtype=e, rank=len(row), flags=0, dims=dims,
                                           key=k.encode(), key_len=len(k), packed_len=0))
                        keep_q.append(dims)
                        r0[k] += row[0]
                    arr_q = (N.Tensor * len(ts))(*ts)
                    keep_q.append(arr_q)
                    reqs_q.append(N.Request(model_name=b"m", model_name_len=1, has_version=1, order=N.ORDER_UPB, version=1, n_inputs=len(ts),
                                            flags=0, inputs=arr_q))
                return (N.Request * n)(*reqs_q), keep_q

            reqs0, keep0 = plan_quo({k: s.cpu().numpy().reshape(n, -1) for k, s in S.items()})
            qcap = C.c_uint64()
            N.check(lib.b200tfs_request_arena_size(n, reqs0, C.byref(qcap)))
            qcap.value += 4096 * n      # b200tfs_encode_requests_async gives every record a worst-case slot: room for its prefix bound
            qmem = C.c_void_p()
            N.check(lib.b200tfs_malloc(qc.ctx, qcap.value + 256, C.byref(qmem)))
            qarena = (qmem.value + 255) & ~255

            def quo():
                sh = {k: s.cpu().numpy().reshape(n, -1) for k, s in S.items()}      # D2H of the shapes + a synchronise
                reqs_q, keep_q = plan_quo(sh)
                N.check(lib.b200tfs_encode_requests_async(qc.ctx, n, reqs_q, qarena, qcap.value))
                qc.sync()

            def existing():                                                          # the same encode, planned once: kernels only
                N.check(lib.b200tfs_encode_requests_async(qc.ctx, n, reqs0, qarena, qcap.value))
                qc.sync()

            res["quo"], _ = timed(quo, reps)
            res["existing"], _ = timed(existing, reps)
            N.check(lib.b200tfs_encode_results(qc.ctx, n, off, ln))
            end = max(int(off[i]) + int(ln[i]) for i in range(n))
            host = np.empty(end, np.uint8)
            N.check(lib.b200tfs_memcpy_d2h(qc.ctx, host.ctypes.data, qarena, end))
            qc.sync()
            assert [host[off[i]: off[i] + ln[i]].tobytes() for i in range(n)] == wires, f"{name}: status-quo bytes differ"
            N.check(lib.b200tfs_free(qc.ctx, qmem.value))
            qc.close()
        host_in = {k: t.cpu().numpy() for k, t in inputs.items()}
        dt_def, dw = timed(lambda: codec._padded_requests_on_host("m", 1, host_in, {k: s.cpu().numpy() for k, s in S.items()}, {}, n), 1)
        assert dw == wires, f"{name}: definition bytes differ"
        res["defn"] = dt_def
        line = {"workload": name, "n": n, "src_bytes": src, "wire_bytes": wire_bytes}
        for leg, t in res.items():
            gbs = (src + wire_bytes) / t / 1e9
            line[leg] = {"ms": round(t * 1e3, 3), "GB/s": round(gbs, 1), "share": round(gbs / 3350, 3)}
        print(json.dumps(line))
        out["workloads"][name] = line
        del inputs, S
        torch.cuda.empty_cache()
    if args:      # a JSON copy of the lines
        with open(args[0], "w") as f:
            json.dump(out, f, indent=1)
    codec.close()


if __name__ == "__main__":
    main()
