#!/usr/bin/env python
"""Throughput of the packed-varint paths (int_val / int64_val ...) on one GPU, for a few value
distributions.  Numbers for DESIGN.md; not the bench line.

    python tools/varint_probe.py [--elems 16777216] [--reps 5] [--only mixed]
    python tools/varint_probe.py --responses [--reps 50]     # varint outputs of 256 PredictResponses, two-phase vs one launch
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(REPO, "min-tfs-client_b200"), os.path.join(REPO, "tests"), REPO, os.path.join(REPO, "tools")]
from batch_probe import timed  # noqa: E402
from devutil import Dev  # noqa: E402
from min_tfs_client import _native as N  # noqa: E402


def cases(m, rng):
    yield "token_ids_int64", 9, rng.integers(0, 50000, size=m, dtype=np.int64)
    mixed = (rng.integers(0, 2 ** 62, size=m, dtype=np.int64) >> rng.integers(0, 62, size=m)).astype(np.int64)
    mixed[::7] *= -1
    yield "mixed_int64", 9, mixed
    yield "int32_signed", 3, rng.integers(-1000, 100000, size=m, dtype=np.int64).astype(np.int32)
    yield "uint8", 4, rng.integers(0, 256, size=m, dtype=np.int64).astype(np.uint8)


def card():
    """Name and power limit of GPU 0, read in the same run as the numbers."""
    import subprocess
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip() or "unknown"


def responses_leg(reps):
    """256 (and 4096 small) PredictResponses with an int64 output and a float32 one, decoded (a) the two-phase way for the varint output -
    single-launch decode + b200tfs_decode_results + b200tfs_unpack_outputs - and (b) by the single-launch decode with
    b200tfs_set_decode_varints on, eagerly and as a captured graph.  Times are CUDA events over `reps` calls."""
    from oracle import wire_oracle
    K = N.FUSED_MAX_OUTPUTS
    rng = np.random.default_rng(0)
    # the last case is the planner's worst kind of batch: many small records (one CTA plans every (record, output) slot)
    shapes = {"tokens": ((8, 512), 256), "classes": ((8, 5), 256), "classes_x4096": ((8, 5), 4096)}
    res = {"card": card()}
    for name, (shp, n) in shapes.items():
        recs = [wire_oracle.build_predict_response([("ids", rng.integers(0, 50000, shp).astype(np.int64)),
                                                    ("scores", rng.standard_normal(shp).astype(np.float32))]) for _ in range(n)]
        offs, cur = [], 0
        for r in recs:
            offs.append(cur)
            cur = (cur + len(r) + 255) & ~255
        arena = np.zeros(cur, dtype=np.uint8)
        for o, r in zip(offs, recs):
            arena[o: o + len(r)] = np.frombuffer(r, dtype=np.uint8)
        off, ln = (C.c_uint64 * n)(*offs), (C.c_uint64 * n)(*[len(r) for r in recs])
        ne = int(np.prod(shp))
        stride = (max(len(r) for r in recs) + 8 * ne + 256 * (K + 1) + 255) & ~255
        wire_bytes = sum(len(r) for r in recs)
        alg = wire_bytes + n * ne * (8 + 4)            # wire read once, both outputs written
        legs = {}
        for mode in ("two_phase", "varints_eager", "varints_graph"):
            dev = Dev(0)
            lib = dev.lib
            a = dev.upload(arena)
            dst = dev.malloc(n * stride)
            ids = dev.malloc(n * ne * 8)
            outs, n_outs, specs, st = (N.Output * (n * K))(), (C.c_int32 * n)(), (N.ModelSpec * n)(), (C.c_int32 * n)()
            N.check(lib.b200tfs_set_decode_varints(dev.ctx, int(mode != "two_phase")))
            ptrs = (C.c_void_p * n)(*[ids + i * ne * 8 for i in range(n)])
            vst = (C.c_int32 * n)()

            def eager():
                N.check(lib.b200tfs_decode_responses(dev.ctx, a, n, off, ln, dst, stride))
                N.check(lib.b200tfs_decode_results(dev.ctx, n, outs, n_outs, specs, st))
                if mode == "two_phase":
                    o_ids = (N.Output * n)(*[outs[i * K] for i in range(n)])
                    N.check(lib.b200tfs_unpack_outputs(dev.ctx, a, n, o_ids, off, ptrs, None, vst))
            eager()
            fn = eager
            if mode == "varints_graph":
                dev.sync()
                N.check(lib.b200tfs_capture_begin(dev.ctx))
                N.check(lib.b200tfs_decode_responses(dev.ctx, a, n, off, ln, dst, stride))
                g = C.c_void_p()
                N.check(lib.b200tfs_capture_end(dev.ctx, C.byref(g)))

                def fn():
                    N.check(lib.b200tfs_graph_launch(dev.ctx, g))
                    N.check(lib.b200tfs_decode_results(dev.ctx, n, outs, n_outs, specs, st))
            t, wall = timed(dev, fn, reps)
            # the routes agree: int64 ids bit for bit
            got = []
            for i in range(n):
                o = outs[i * K]
                assert st[i] == 0 and o.status == 0, (mode, i)
                if mode == "two_phase":
                    got.append(dev.download(ids + i * ne * 8, ne * 8).tobytes())
                else:
                    got.append(dev.download(dst + i * stride + int(o.dst_off), ne * 8).tobytes())
            legs[mode] = {"us": t * 1e6, "wall_us": wall * 1e6, "GBs": alg / t / 1e9, "ids": got}
            dev.close()
        assert legs["two_phase"]["ids"] == legs["varints_eager"]["ids"] == legs["varints_graph"]["ids"]
        for v in legs.values():
            v.pop("ids")
        res[name] = {"responses": n, "wire_bytes": wire_bytes, "decoded_bytes": n * ne * 12, **legs}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--elems", type=int, default=16 << 20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--only", default="")
    ap.add_argument("--responses", action="store_true", help="the varint outputs of the single-launch decode instead (b200tfs_set_decode_varints)")
    args = ap.parse_args()
    if args.responses:
        print(json.dumps(responses_leg(max(args.reps, 20)), indent=1))
        return
    dev = Dev(0)
    lib = dev.lib
    peak = 3350.0      # H100 SXM data sheet, when no measured copy rate is at hand
    try:
        peak = json.load(open(os.path.join(REPO, "MEASURED_PEAKS.json")))["hbm_gbs"]
    except Exception:
        pass
    out = {"elems": args.elems, "peak_GBs": peak}
    rng = np.random.default_rng(0)
    for name, dt, vals in cases(args.elems, rng):
        if args.only and args.only not in name:
            continue
        m = vals.size
        src_bytes = vals.nbytes
        v = dev.upload(vals)
        vd = (C.c_int64 * 1)(m)
        vt = (N.Tensor * 1)(N.Tensor(data=v, src_dtype=dt, wire_dtype=dt, rank=1, flags=0, dims=vd, key=b"", key_len=0, packed_len=0))
        N.check(lib.b200tfs_measure(dev.ctx, 1, vt))
        packed = int(vt[0].packed_len)
        need = C.c_uint64()
        N.check(lib.b200tfs_tensor_arena_size(1, vt, C.byref(need)))
        arena = dev.malloc(need.value)
        o, ln = (C.c_uint64 * 1)(), (C.c_uint64 * 1)()
        alg = src_bytes + packed

        def both():
            N.check(lib.b200tfs_measure(dev.ctx, 1, vt))
            N.check(lib.b200tfs_encode_tensor_protos(dev.ctx, 1, vt, arena, need.value, o, ln))
        t_me, _ = timed(dev, both, args.reps)
        t_m, _ = timed(dev, lambda: N.check(lib.b200tfs_measure(dev.ctx, 1, vt)), args.reps)
        t_e, _ = timed(dev, lambda: N.check(lib.b200tfs_encode_tensor_protos(dev.ctx, 1, vt, arena, need.value, o, ln)), args.reps)
        # the deferred encode: the same tensor as the only input of a PredictRequest, packed_len unset - no host round trip; the
        # count -> frame -> emit
        vt2 = (N.Tensor * 1)(N.Tensor(data=v, src_dtype=dt, wire_dtype=dt, rank=1, flags=0, dims=vd, key=b"ids", key_len=3, packed_len=0))
        rq = (N.Request * 1)(N.Request(model_name=b"m", model_name_len=1, has_version=0, order=N.ORDER_UPB, version=0, n_inputs=1, flags=0, inputs=vt2))
        need2 = C.c_uint64()
        N.check(lib.b200tfs_request_arena_size(1, rq, C.byref(need2)))
        arena_d = dev.malloc(need2.value)
        t_def, _ = timed(dev, lambda: N.check(lib.b200tfs_encode_requests_async(dev.ctx, 1, rq, arena_d, need2.value)), args.reps)
        do, dl = (C.c_uint64 * 1)(), (C.c_uint64 * 1)()
        N.check(lib.b200tfs_encode_results(dev.ctx, 1, do, dl))
        got = dev.download(arena_d + int(do[0]), int(dl[0]))
        ref = dev.download(arena + int(o[0]), int(ln[0]))
        assert got[-packed:].tobytes() == ref[-packed:].tobytes() and int(dl[0]) > packed      # same packed payload as the measured encode
        outs = (N.Output * 1)()
        st = (C.c_int32 * 1)()
        N.check(lib.b200tfs_parse_tensor_protos(dev.ctx, arena, 1, o, ln, outs, st))
        assert st[0] == 0 and outs[0].n_elems == m
        back = dev.malloc(src_bytes)
        dptr = (C.c_void_p * 1)(back)
        t_d, _ = timed(dev, lambda: N.check(lib.b200tfs_unpack_outputs(dev.ctx, arena, 1, outs, o, dptr, None, None)), args.reps)
        assert np.array_equal(dev.download(back, src_bytes).view(vals.dtype), vals)
        out[name] = {"src_bytes": src_bytes, "packed_bytes": packed,
                     "measure_us": t_m * 1e6, "encode_us": t_e * 1e6, "measure_plus_encode_us": t_me * 1e6, "decode_us": t_d * 1e6,
                     "deferred_encode_us": t_def * 1e6, "deferred_encode_frac": alg / t_def / 1e9 / peak,
                     "encode_frac": alg / t_me / 1e9 / peak, "encode_only_frac": alg / t_e / 1e9 / peak, "decode_frac": alg / t_d / 1e9 / peak}
    print(json.dumps(out, indent=1))
    dev.close()


if __name__ == "__main__":
    main()
