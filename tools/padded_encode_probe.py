"""Time Codec.encode_predict_requests_padded / b200tfs_encode_padded_requests_async against the status quo, and compare every leg's
bytes after its timed region.

Workloads (sequence and image clients whose batch is already on the GPU):
  U1  1024 x {input_ids, attention_mask: int64[1, T_r]} from int64[1024, 512], T_r in 16..512, ids in 0..50000
  U2  256 x f32[1, T_r, 1024] from f32[256, 512, 1024]
  U3  the split of f32[262144, 1024] into 256 x f32[1024, 1024]
  U4  64 x f32[1, H_r, W_r, 3] from f32[64, 512, 512, 3]
Legs:
  device  the C call, eager (host call to results, arena ready on the device) and as a replayed CUDA graph
  quo     the status quo: shapes to the host, a synchronise, per-request structs over the device boxes planned on the host, then
          b200tfs_encode_requests_async; the wire stays on the device, as in the device legs (contiguous boxes only: U1-U3)
  existing  the same b200tfs_encode_requests_async with the requests planned once: the existing encode at equal bytes
  python  Codec.encode_predict_requests_padded (bytes on the host)
  defn    the definition: host slicing, then encode_predict_requests
Usage: python tools/padded_encode_probe.py [out.json]
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
sys.path[:0] = [os.path.join(HERE, "..", "min-tfs-client_b200"), os.path.join(HERE, "..")]

import torch  # noqa: E402

from min_tfs_client import _native as N  # noqa: E402
from min_tfs_client.codec import Codec  # noqa: E402


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


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("card:", q)
    codec = Codec(0)
    lib = N.load()
    rng = np.random.default_rng(0)
    out = {"card": q, "workloads": {}}
    for name, inputs, shapes, contiguous in workloads(rng):
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
    if len(sys.argv) > 1:      # a JSON copy of the lines
        with open(sys.argv[1], "w") as f:
            json.dump(out, f, indent=1)
    codec.close()


if __name__ == "__main__":
    main()
