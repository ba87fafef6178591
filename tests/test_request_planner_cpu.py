"""The PredictRequest planners' host entry points, pinned: the immediate planner (b200tfs_request_frame, b200tfs_request_size,
b200tfs_request_arena_size on measured batches) and the deferred one (b200tfs_request_arena_size on unmeasured batches,
b200tfs_request_frame_deferred) against what they returned when these pins were written, byte for byte, over the request
goldens and a seeded random corpus; and the status each of them returns on a table of malformed requests.

`python tests/test_request_planner_cpu.py` rewrites tests/golden/request_planner.json from the library as built.  Do that only
for a change that means to alter the framing."""
import ctypes as C
import functools
import hashlib
import json
import os

import numpy as np
import pytest

import golden_util as G
from min_tfs_client import _native as N
from min_tfs_client.codec import _Prepared

PINS = "request_planner.json"
MULTS = (1, 5, 10)          # b200tfs_request_frame_deferred: packed lengths at this many bytes per element
DTYPES = [np.float32, np.float64, np.int32, np.uint8, np.int16, np.int8, np.complex64, np.int64, np.bool_, np.uint16,
          np.complex128, np.float16, np.uint32, np.uint64, "bfloat16"]


def _packed_len(t, arr):
    """Bytes of the packed-varint payload of a prepared tensor, 0 when its values are not packed varints."""
    if t.flags & (N.F_TENSOR_CONTENT | N.F_PRESERIALIZED) or t.src_dtype != t.wire_dtype or arr.size == 0:
        return 0
    if arr.dtype.itemsize == 2 and arr.dtype.kind not in "iu":              # DT_HALF / DT_BFLOAT16: half_val bit patterns
        u = arr.view(np.uint16).astype(np.uint64)
    elif arr.dtype.kind in "iu":
        u = arr.astype(np.int64).view(np.uint64) if arr.dtype.kind == "i" else arr.astype(np.uint64)   # negatives: ten bytes
    else:
        return 0
    return int(sum((u >= np.uint64(1 << (7 * k))).sum() for k in range(1, 10))) + arr.size


class Req:
    """One request in two states: varint inputs measured (packed_len set) and unmeasured (packed_len 0)."""

    def __init__(self, name, version, inputs, order=N.ORDER_UPB, grpc=False):
        self.preps = [_Prepared(a, k, wd, content, snan) for k, a, wd, content, snan in inputs]
        self.packed = [_packed_len(p.struct, p.array) for p in self.preps]
        self.name = name
        n = max(len(self.preps), 1)
        self.measured = (N.Tensor * n)(*[p.struct for p in self.preps])
        self.unmeasured = (N.Tensor * n)(*[p.struct for p in self.preps])
        for i, pl in enumerate(self.packed):
            self.measured[i].packed_len = pl
        self.req = {m: N.Request(model_name=name, model_name_len=len(name), has_version=int(version is not None), order=order,
                                 version=version or 0, n_inputs=len(self.preps), flags=N.RF_GRPC_FRAME if grpc else 0,
                                 inputs=self.measured if m else self.unmeasured) for m in (True, False)}


def _digest(*parts):
    h = hashlib.sha256()
    for p in parts:
        h.update(p if isinstance(p, bytes) else repr(p).encode())
    return h.hexdigest()[:20]


def frame(lib, req, n):
    m = max(n, 1)
    buf = C.create_string_buffer(1 << 16)
    flen = C.c_uint64()
    poff, plen, perm = (C.c_uint64 * m)(), (C.c_uint64 * m)(), (C.c_int32 * m)()
    rc = lib.b200tfs_request_frame(C.byref(req), buf, 1 << 16, C.byref(flen), poff, plen, perm)
    if rc:
        return rc, ""
    return rc, _digest(buf.raw[: flen.value], list(poff[:n]), list(plen[:n]), list(perm[:n]))


def size(lib, req):
    total = C.c_uint64()
    rc = lib.b200tfs_request_size(C.byref(req), C.byref(total))
    return rc, (str(total.value) if rc == 0 else "")


def arena(lib, req):
    need = C.c_uint64()
    rc = lib.b200tfs_request_arena_size(1, C.byref(req), C.byref(need))
    return rc, need.value


def deferred(lib, req, n, packed, cap):
    m = max(n, 1)
    buf = np.zeros(cap, np.uint8)
    pk = (C.c_uint64 * m)(*packed[:m])
    off, ln = C.c_uint64(), C.c_uint64()
    poff, plen = (C.c_uint64 * m)(), (C.c_uint64 * m)()
    rc = lib.b200tfs_request_frame_deferred(C.byref(req), pk, buf.ctypes.data, cap, C.byref(off), C.byref(ln), poff, plen)
    if rc:
        return rc, ""
    return rc, _digest(off.value, ln.value, buf.tobytes(), list(poff[:n]), list(plen[:n]))


def outputs(r):
    """Every planner entry point on one request: {entry point: "status digest"}."""
    lib = N.load()
    n = len(r.preps)
    out = {"frame": frame(lib, r.req[True], n), "size": size(lib, r.req[True])}
    rc, need = arena(lib, r.req[True])
    out["arena_measured"] = (rc, str(need) if rc == 0 else "")
    rc, need = arena(lib, r.req[False])
    out["arena_unmeasured"] = (rc, str(need) if rc == 0 else "")
    cap = (need if rc == 0 else 0) + 4096      # room for the deferred worst case of a batch without unmeasured inputs
    for k in MULTS:
        out["deferred_%d" % k] = deferred(lib, r.req[False], n, [k * p.size for p in r.preps], cap)
    return {ep: "%d %s" % v for ep, v in out.items()}


# ---- corpus ---------------------------------------------------------------------------------------------------------------
def golden_requests():
    cases = {}
    for name, case in G.load("requests.json").items():
        wd = case.get("wire_dtype")
        inputs = [(k.encode(), G.make_array(rec), wd, False, False) for k, rec in case["inputs"]]
        cases["golden:" + name] = lambda n=case["model_name"], v=case["model_version"], i=inputs: Req(n.encode(), v, i)
    return cases


def _array(rng, dt):
    rank = int(rng.integers(0, 5))
    shape = [int(rng.integers(0, 6)) for _ in range(rank)]
    if rank and rng.random() < 0.15:
        shape[0] = int(rng.choice([33, 200, 700]))        # past the tiny-varint count, the warp path's 2 KB, a 2-byte dim
    if dt == "bfloat16":
        import ml_dtypes

        return rng.standard_normal(shape).astype(ml_dtypes.bfloat16)
    dt = np.dtype(dt)
    if dt.kind == "b":
        return rng.integers(0, 2, size=shape).astype(np.bool_)
    if dt.kind in "iu":
        info = np.iinfo(dt)
        return rng.integers(info.min, info.max, size=shape, dtype=dt, endpoint=True)
    if dt.kind == "c":
        return (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).astype(dt)
    return rng.standard_normal(shape).astype(dt)


def _key(rng, used):
    while True:
        k = bytes(rng.choice([97, 98, 66, 0, 255, 0xC3], size=int(rng.integers(0, 5))).astype(np.uint8))
        if rng.random() < 0.05:
            k = k + b"k" * 140                              # a key whose length prefix takes two bytes
        if k not in used:
            used.add(k)
            return k


def random_request(seed):
    rng = np.random.default_rng([20261017, seed])
    used = set()
    n_in = int(rng.choice([0, 1, 1, 2, 3, 4, 5, 18]))      # 18: more keys than the planner keeps inline
    inputs = []
    for _ in range(n_in):
        kind = rng.random()
        key = _key(rng, used)
        if kind < 0.08:                                     # DT_STRING: a pre-serialised TensorProto
            shape = [int(rng.integers(0, 4)) for _ in range(int(rng.integers(0, 3)))]
            words = np.array(["w" * int(rng.integers(0, 9)) for _ in range(int(np.prod(shape)))], dtype=np.str_).reshape(shape)
            inputs.append((key, words, None, False, False))
            continue
        dt = DTYPES[int(rng.integers(0, len(DTYPES)))]
        a = _array(rng, dt)
        half = dt in (np.float16, "bfloat16")
        wd = "DT_FLOAT" if half and rng.random() < 0.4 else None
        inputs.append((key, a, wd, bool(rng.random() < 0.2), bool(dt is np.float32 and rng.random() < 0.3)))
    name = bytes(rng.choice([109, 0xC3, 0xA8], size=int(rng.choice([0, 1, 7, 130]))).astype(np.uint8))
    version = [None, 0, 1, 300, 1 << 40, -1][int(rng.integers(0, 6))]
    order = int(rng.integers(0, 3))
    return Req(name, version, inputs, order=order, grpc=bool(rng.random() < 0.4))


def corpus():
    cases = golden_requests()
    for s in range(240):
        cases["random:%d" % s] = lambda s=s: random_request(s)
    return cases


CORPUS = corpus()


@functools.lru_cache(maxsize=None)
def _pins():
    return G.load(PINS)


@pytest.mark.parametrize("case", list(CORPUS))
def test_planners_give_the_pinned_framing(case):
    pin = _pins()[case]
    assert outputs(CORPUS[case]()) == pin, case


def test_corpus_reaches_every_state():
    """The corpus exercises what the planners branch on: every dtype, casts, tensor_content, pre-serialised inputs, empty and
    rank-0 tensors, tiny and large packed-varint inputs, each key order, the gRPC frame - and the pins say OK for them."""
    seen = set()
    for name, make in CORPUS.items():
        r = make()
        q = r.req[True]
        seen.add(("order", q.order))
        seen.add(("grpc", q.flags))
        seen.add(("many keys", q.n_inputs > 16))
        for p, pl in zip(r.preps, r.packed):
            t = p.struct
            seen.add(("dtype", t.src_dtype))
            seen.add(("rank", min(t.rank, 4)))
            seen.add(("empty", p.size == 0))
            seen.add(("flags", t.flags))
            seen.add(("cast", t.src_dtype != t.wire_dtype))
            if pl:
                seen.add(("varint", "tiny" if p.size <= 32 else "large"))
    want = {("order", o) for o in range(3)} | {("grpc", 0), ("grpc", 1), ("many keys", True)} | {("rank", k) for k in range(5)}
    want |= {("dtype", d) for d in (1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 14, 17, 18, 19, 22, 23)} | {("empty", True), ("cast", True)}
    want |= {("flags", f) for f in (0, N.F_TENSOR_CONTENT, N.F_KEEP_SNAN, N.F_PRESERIALIZED)} | {("varint", "tiny"), ("varint", "large")}
    assert want <= seen, want - seen
    pins = _pins()
    for ep in ("frame", "size", "arena_measured", "arena_unmeasured", "deferred_1", "deferred_10"):
        assert sum(1 for c in CORPUS if pins[c][ep].startswith("0 ")) > 150, ep


# ---- malformed requests ---------------------------------------------------------------------------------------------------
def _base():
    """img float32 (2, 3), ids int64 (40,) - a packed-varint input past the tiny count - and mask bool (5,)."""
    return Req(b"m", 3, [(b"img", np.arange(6, dtype=np.float32).reshape(2, 3), None, False, False),
                         (b"ids", np.arange(40, dtype=np.int64) - 20, None, False, False),
                         (b"mask", np.ones(5, np.bool_), None, False, False)])


def _dims(*d):
    return (C.c_int64 * len(d))(*d)


def _set(i, **kw):
    def mutate(r, ts, keep):
        for f, v in kw.items():
            setattr(ts[i], f, v)
    return mutate


def _req(**kw):
    def mutate(r, ts, keep):
        for f, v in kw.items():
            setattr(r, f, v)
    return mutate


def _both(*ms):
    def mutate(r, ts, keep):
        for m in ms:
            m(r, ts, keep)
    return mutate


def _unaligned(r, ts, keep):
    ts[1].data += 1


def _preserialized_2g(r, ts, keep):
    ts[2].flags, ts[2].rank, ts[2].packed_len = N.F_PRESERIALIZED, 0, 1 << 31


def _varint_16g(r, ts, keep):
    keep.append(_dims(1 << 33))
    ts[1].dims = keep[-1]
    if ts[1].packed_len:
        ts[1].packed_len = 1 << 34


# status of (frame, size, arena, deferred frame) on the measured request, then the same four on the unmeasured one
E_ARG, E_SHAPE, E_DTYPE, E_TOOBIG, E_SIZE, OK = N.E_ARG, N.E_SHAPE, N.E_DTYPE, N.E_TOOBIG, N.E_SIZE, N.OK
MALFORMED = {
    "well_formed": (None, (OK, OK, OK, OK, E_ARG, E_ARG, OK, OK)),
    "negative_n_inputs": (_req(n_inputs=-1), (E_ARG, E_ARG, E_ARG, E_ARG, E_ARG, E_ARG, E_ARG, E_ARG)),
    "null_inputs": (_req(inputs=None), (E_ARG, E_ARG, E_ARG, E_ARG, E_ARG, E_ARG, E_ARG, E_ARG)),
    "negative_model_name_len": (_req(model_name_len=-1), (E_ARG, E_ARG, E_ARG, E_ARG, E_ARG, E_ARG, E_ARG, E_ARG)),
    "null_model_name": (_req(model_name=None), (E_ARG, E_ARG, E_ARG, E_ARG, E_ARG, E_ARG, E_ARG, E_ARG)),
    "unknown_flags": (_req(flags=0x6), (E_ARG, E_ARG, E_ARG, E_ARG, E_ARG, E_ARG, E_ARG, E_ARG)),
    "unknown_key_order": (_req(order=9), (E_ARG, E_ARG, E_ARG, E_ARG, E_ARG, E_ARG, E_ARG, E_ARG)),
    "negative_key_len": (_set(0, key_len=-1), (E_ARG, E_ARG, E_ARG, E_ARG, E_ARG, E_ARG, E_ARG, E_ARG)),
    "null_key": (_set(1, key=None), (E_ARG, E_ARG, E_ARG, E_ARG, E_ARG, E_ARG, E_ARG, E_ARG)),
    "negative_dim": (_set(0, dims=_dims(2, -3)), (E_SHAPE, E_SHAPE, E_SHAPE, E_SHAPE, E_ARG, E_ARG, E_SHAPE, E_SHAPE)),
    "null_dims_fixed_width": (_set(0, dims=None), (E_ARG, E_ARG, E_ARG, E_SHAPE, E_ARG, E_ARG, E_SHAPE, E_SHAPE)),
    "null_dims_varint": (_set(1, dims=None), (E_ARG, E_ARG, E_ARG, E_SHAPE, E_ARG, E_ARG, E_ARG, E_SHAPE)),
    "rank_over_254": (_set(0, rank=300), (E_SHAPE, E_SHAPE, E_SHAPE, E_SHAPE, E_ARG, E_ARG, E_SHAPE, E_SHAPE)),
    "negative_rank": (_set(2, rank=-1), (E_SHAPE, E_SHAPE, E_SHAPE, E_SHAPE, E_ARG, E_ARG, E_SHAPE, E_SHAPE)),
    "string_wire_dtype": (_set(0, src_dtype=7, wire_dtype=7), (E_DTYPE, E_DTYPE, E_DTYPE, E_DTYPE, E_ARG, E_ARG, E_DTYPE, E_DTYPE)),
    "unknown_dtype": (_set(2, src_dtype=99, wire_dtype=99), (E_DTYPE, E_DTYPE, E_DTYPE, E_DTYPE, E_ARG, E_ARG, E_DTYPE, E_DTYPE)),
    "unsupported_cast": (_set(0, src_dtype=2), (E_DTYPE, E_DTYPE, E_DTYPE, E_DTYPE, E_ARG, E_ARG, E_DTYPE, E_DTYPE)),
    "null_data_fixed_width": (_set(0, data=None), (OK, OK, OK, E_ARG, E_ARG, E_ARG, E_ARG, E_ARG)),
    "null_data_varint": (_set(1, data=None), (OK, OK, OK, E_ARG, E_ARG, E_ARG, E_ARG, E_ARG)),
    "unaligned_varint_data": (_unaligned, (OK, OK, OK, E_ARG, E_ARG, E_ARG, E_ARG, E_ARG)),
    "tensor_over_2g": (_set(0, dims=_dims(1 << 20, 1 << 12)), (E_TOOBIG, E_TOOBIG, E_TOOBIG, E_TOOBIG, E_ARG, E_ARG, E_TOOBIG, E_TOOBIG)),
    "element_count_overflow": (_set(0, dims=_dims(1 << 40, 1 << 40)), (E_TOOBIG, E_TOOBIG, E_TOOBIG, E_TOOBIG, E_ARG, E_ARG, E_TOOBIG, E_TOOBIG)),
    "varint_over_2g": (_varint_16g, (E_TOOBIG, E_TOOBIG, E_TOOBIG, E_TOOBIG, E_ARG, E_ARG, E_TOOBIG, E_TOOBIG)),
    "preserialized_over_2g": (_preserialized_2g, (E_TOOBIG, E_TOOBIG, E_TOOBIG, E_TOOBIG, E_ARG, E_ARG, E_TOOBIG, E_TOOBIG)),
    "request_over_2g": (_both(_set(0, rank=1, dims=_dims(3 << 27)), _set(2, dims=_dims(3 << 29))), (E_TOOBIG, E_TOOBIG, E_TOOBIG, E_SIZE, E_ARG, E_ARG, OK, E_SIZE)),
}


def malformed_codes(mutate):
    lib = N.load()
    codes = []
    for measured in (True, False):
        r = _base()
        q, ts, keep = r.req[measured], (r.measured if measured else r.unmeasured), []
        if mutate:
            mutate(q, ts, keep)
        n = len(r.preps)
        codes += [frame(lib, q, n)[0], size(lib, q)[0], arena(lib, q)[0], deferred(lib, q, 8, [40] * 8, 1 << 16)[0]]
    return tuple(codes)


@pytest.mark.parametrize("case", list(MALFORMED))
def test_malformed_requests_keep_their_status(case):
    mutate, want = MALFORMED[case]
    assert malformed_codes(mutate) == want, case


if __name__ == "__main__":
    pins = {c: outputs(make()) for c, make in CORPUS.items()}
    with open(os.path.join(G.GOLDEN_DIR, PINS), "w") as fh:
        json.dump({"cases": pins}, fh, indent=0, sort_keys=True)
        fh.write("\n")
    print("wrote %d pins" % len(pins))
