"""Which route every Python decode call takes, pinned case by case.

For every case below - float, varint, string and mixed outputs, more than eight outputs, malformed records, TF padding,
tensor_content, strict DT_HALF, ``out_dtypes`` narrowing, pinned and ordinary ``out=``, ``open_predict_response`` +
``OpenResponse.array`` and the concatenated and padded decodes - the test records what comes back (dtype, shape and a digest
of the bytes, or the exception type), whether each returned array is a view of the launch's host buffer, a fresh array or the
caller's ``out=`` array, how far ``kernel_launches()``, ``concat_device_calls`` and ``b200tfs_decode_stats`` advance, and how
many times each native decode entry point runs.  Each case runs twice on a fresh codec, and twice again on a codec that has
already seen varint outputs (``_seen_varints``), so that the templates the first call leaves and the varint switch are
pinned as well.  EXPECTED is what the codec did when the routes were last changed on purpose: a route that changes shows
up here first.
"""
import ctypes as C
import hashlib
import json

import ml_dtypes
import numpy as np
import pytest

import decode_mutants as D
from min_tfs_client import _native as N
from min_tfs_client import device as DV
from min_tfs_client.codec import Codec, DecodedSpec
from oracle import wire_oracle

pytestmark = pytest.mark.gpu

COUNTED = ("b200tfs_decode_responses_host_async", "b200tfs_decode_results", "b200tfs_parse_responses_host",
           "b200tfs_parse_tensor_protos_host", "b200tfs_unpack_outputs_host", "b200tfs_unpack_outputs", "b200tfs_set_decode_cast",
           "b200tfs_set_decode_varints", "b200tfs_decode_slot_bytes", "b200tfs_response_keys", "b200tfs_concat_layout",
           "b200tfs_decode_concat", "b200tfs_concat_results", "b200tfs_padded_layout", "b200tfs_decode_padded",
           "b200tfs_padded_results", "b200tfs_memcpy_h2d", "b200tfs_memcpy_d2h")

build = wire_oracle.build_predict_response
rng = np.random.default_rng(20261016)
F32, F64 = rng.standard_normal((8, 5)).astype(np.float32), rng.standard_normal(3)
Y = rng.standard_normal((64, 33)).astype(np.float32)
IDS = rng.integers(-5, 50000, (3, 7)).astype(np.int64)

FLOATS = build([("scores", F32), ("d", F64)])
FLOATS2 = build([("scores", F32 * 2), ("d", F64 - 1)])
ONE = build([("y", Y)])
VARINT = build([("ids", IDS), ("mask", rng.integers(0, 2, 9).astype(bool)), ("small", rng.integers(-9, 9, 5).astype(np.int32))])
VARINT1 = build([("ids", IDS[0])])
MIXED = build([("classes", rng.integers(0, 1000, (8, 5)).astype(np.int64)), ("scores", F32), ("d", F64.reshape(3, 1))])
MIXED2 = build([("classes", rng.integers(0, 1000, (2, 5)).astype(np.int64)), ("scores", F32[:2]), ("d", F64[:1].reshape(1, 1))])
HALF = build([("h", rng.standard_normal(6).astype(np.float16)), ("f", F32[0])])
CONTENT = build([("c", F32)], tensor_content=True)
MANY = build([(f"o{i}", F32[i % 8] + i) for i in range(9)])
MANY_MIXED = build([(f"o{i}", F32[i % 8] if i % 2 else IDS[i % 3]) for i in range(10)])
RANK0 = build([("r", np.float32(2.5).reshape(()))])
NARROW = build([("f", rng.standard_normal((30, 7)).astype(np.float32)), ("g", rng.standard_normal(99).astype(np.float32)),
                ("ids", rng.integers(0, 1000, 50))])
NARROW_F = build([("f", rng.standard_normal((30, 7)).astype(np.float32)), ("g", rng.standard_normal(99).astype(np.float32))])
SEEDS = {s.name: s.wire for s in D.seeds()}
STRINGS, TF_CONTENT = SEEDS["multi"], SEEDS["content"]
PAD = D.out("p", 1, [6], D.ld(0x2A, D.f32(2, 1).tobytes())) + D.out("z", 1, [4], b"") + D.mspec()
BF16 = D.out("b", 14, [2], D.ld(0x6A, D.packed_varints([16256, 0]))) + D.mspec()
CPLX = D.out("c", 8, [2], D.ld(0x4A, D.f32(4, 2).tobytes())) + D.mspec()
VARINT_BAD = {
    "few": D.out("x", 9, [4], D.ld(0x52, D.packed_varints([1, 2, 3]))) + D.mspec(),
    "parse": D.out("x", 9, [4], D.ld(0x52, D.packed_varints([1, 2]) + b"\xff" * 10 + b"\x01")) + D.mspec(),
    "range": D.out("x", 6, [3], D.ld(0x3A, D.packed_varints([1, 2, 300]))) + D.mspec(),
    "rows": D.out("x", 3, [3], b"".join(D.vi(7 << 3) + D.vi(v) for v in (5, 6, 7))) + D.mspec(),
    "half": D.out("x", 19, [2], D.ld(0x6A, D.packed_varints([18688, 1]))) + D.mspec(),
}
ZERO_RUN = D.out("y", 1, [0], D.ld(0x2A, b"")) + D.mspec()          # an empty packed float_val: one run, no elements
ZERO_VARINT = D.out("v", 9, [0], D.ld(0x52, b"")) + D.mspec()
TRUNCATED = MIXED[: len(MIXED) // 2]
FLIPPED = bytes([FLOATS[0] ^ 0x40]) + FLOATS[1:]
WARM = build([("ids", np.arange(40, dtype=np.int64)), ("s", F32[0])])

SINGLES = {"floats": FLOATS, "one": ONE, "varint": VARINT, "mixed": MIXED, "half": HALF, "content": CONTENT, "many": MANY,
           "many_mixed": MANY_MIXED, "rank0": RANK0, "strings": STRINGS, "tf_content": TF_CONTENT, "pad": PAD, "bf16": BF16,
           "complex": CPLX, "truncated": TRUNCATED, "flipped": FLIPPED, "empty": b"", "zero_run": ZERO_RUN,
           "zero_varint": ZERO_VARINT, "zero_none": build([("y", np.zeros(0, np.float32))]),
           **{"varint_" + k: w for k, w in VARINT_BAD.items()}}


def _decode(wires, **kw):
    return lambda c: (c.decode_predict_responses(wires, **kw), [])


def _pinned_out(wire_pinned=False, strict=False, key="y", wire=ONE, shape=Y.shape, dtype=np.float32, **kw):
    def run(c):
        dst = c.pinned_empty(shape, dtype)
        dst[...] = 0
        w = wire
        if wire_pinned:
            w = c.pinned_empty((len(wire),), np.uint8)
            w[...] = np.frombuffer(wire, np.uint8)
        return c.decode_predict_response(w, out={key: dst}, strict=strict, **kw), [dst]
    return run


def _numpy_out(wire, outs, **kw):
    def run(c):
        dst = {k: np.zeros(s, t) for k, (s, t) in outs.items()}
        return c.decode_predict_response(wire, out=dst, **kw), list(dst.values())
    return run


def _open(wire):
    def run(c):
        opened = c.open_predict_response(wire)
        if opened is None:
            return None, []
        got = {}
        for k in opened.table:
            got[k] = [_outcome(lambda: opened.array(k, strict)) for strict in (False, True, False)]
            got[k].append(hashlib.sha1(opened.wire_of(k)).hexdigest()[:12])
        return got, []
    return run


def _concat(wires, out=None, **kw):
    def run(c):
        dst = {}
        for k, v in (out or {}).items():
            shape, dtype, on_device = v
            dst[k] = c.device_array(np.zeros(shape, dtype)) if on_device else np.zeros(shape, dtype)
        return c.decode_predict_responses_concat(wires, out=dst or None, **kw), list(dst.values())
    return run


def _padded(wires, out=None, **kw):
    """``out`` values: (shape, dtype, where) with where False (numpy), True (device array) or "torch" (a torch tensor 8 bytes
    past a 16-byte boundary: the device route refuses it), returned as a host copy."""
    def run(c):
        dst = {}
        for k, (shape, dtype, where) in (out or {}).items():
            if where == "torch":
                import torch

                dst[k] = torch.from_numpy(np.zeros(int(np.prod(shape)) + 1, dtype)).cuda()[1:].view(*shape)
            else:
                dst[k] = c.device_array(np.zeros(shape, dtype)) if where else np.zeros(shape, dtype)
        res = c.decode_predict_responses_padded(wires, out=dst or None, **kw)
        for k, v in dst.items():
            if not isinstance(v, (np.ndarray, DV.DeviceArray)):
                res[0][k] = v.cpu().numpy()
        return res, [v for v in dst.values() if isinstance(v, (np.ndarray, DV.DeviceArray))]
    return run


RAGGED = build([("scores", F32[:3, :2] + 1), ("d", F64[:2])])
WIDE = build([("scores", Y[:2, :7]), ("d", F64)])

CASES = {}
for name, w in SINGLES.items():
    for strict in (False, True):
        CASES[f"decode_{name}_{'strict' if strict else 'tolerant'}"] = _decode([w], strict=strict)
    CASES[f"open_{name}"] = _open(w)
CASES.update({
    "batch_floats": _decode([FLOATS, FLOATS2, FLOATS]),
    "batch_mixed": _decode([VARINT, MIXED, STRINGS, HALF]),
    "batch_mixed_strict": _decode([VARINT, MIXED, STRINGS, HALF], strict=True),
    "batch_with_many": _decode([FLOATS, MANY]),
    "batch_with_malformed": _decode([FLOATS, TRUNCATED]),
    "narrow_f16_full": _decode([NARROW], out_dtypes={"f": np.float16, "g": np.float16}),
    "narrow_bf16_full": _decode([NARROW_F, NARROW_F], out_dtypes={"f": ml_dtypes.bfloat16, "g": ml_dtypes.bfloat16}),
    "narrow_f16_partial": _decode([NARROW], out_dtypes={"f": np.float16}),
    "narrow_f16_full_strict": _decode([NARROW], out_dtypes={"f": np.float16, "g": np.float16}, strict=True),
    "narrow_f16_and_ids": _decode([NARROW], out_dtypes={"f": np.float16, "g": np.float16, "ids": np.int32}),
    "cast_ids": _decode([NARROW], out_dtypes={"ids": np.int32}),
    "cast_f64": _decode([NARROW_F], out_dtypes={"f": np.float64}),
    "narrow_f16_padding": _decode([PAD], out_dtypes={"p": np.float16, "z": np.float16}),
    "out_pinned": _pinned_out(),
    "out_pinned_strict": _pinned_out(strict=True),
    "out_pinned_wire": _pinned_out(wire_pinned=True),
    "out_pinned_two_outputs": _pinned_out(key="scores", wire=FLOATS, shape=F32.shape),
    "out_pinned_shape_mismatch": _pinned_out(shape=(3,)),
    "out_pinned_dtype_mismatch": _pinned_out(dtype=np.float64),
    "out_pinned_varint": _pinned_out(key="ids", wire=VARINT1, shape=IDS[0].shape, dtype=np.int64),
    "out_pinned_missing_key": _pinned_out(key="nope"),
    "out_pinned_out_dtypes": _pinned_out(shape=Y.shape, dtype=np.float16, out_dtypes={"y": np.float16}),
    "out_pinned_truncated": _pinned_out(wire=ONE[:-7]),
    "out_pinned_zero_run": _pinned_out(wire=ZERO_RUN, shape=(0,)),
    "out_pinned_zero_none": _pinned_out(wire=build([("y", np.zeros(0, np.float32))]), shape=(0,)),
    "out_pinned_f64": _pinned_out(wire=build([("y", F64)]), shape=F64.shape, dtype=np.float64),
    "out_numpy": _numpy_out(MIXED, {"scores": (F32.shape, np.float32), "classes": ((8, 5), np.int64)}),
    "out_numpy_one": _numpy_out(ONE, {"y": (Y.shape, np.float32)}),
    "out_numpy_mismatch": _numpy_out(MIXED, {"scores": ((3,), np.float32)}),
    "out_numpy_missing_key": _numpy_out(MIXED, {"nope": ((3,), np.float32)}),
    "concat_floats": _concat([FLOATS, FLOATS2, FLOATS]),
    "concat_floats_device": _concat([FLOATS, FLOATS2, FLOATS], device=True),
    "concat_mixed": _concat([MIXED, MIXED2]),
    "concat_mixed_device": _concat([MIXED, MIXED2], device=True),
    "concat_mixed_strict": _concat([MIXED, MIXED2], strict=True),
    "concat_keys": _concat([MIXED, MIXED2], keys=["d", "classes"]),
    "concat_strings": _concat([STRINGS, STRINGS]),
    "concat_strings_device": _concat([STRINGS, STRINGS], device=True),
    "concat_half": _concat([HALF, HALF]),
    "concat_half_strict": _concat([HALF, HALF], strict=True),
    "concat_narrow": _concat([NARROW, NARROW], out_dtypes={"f": np.float16, "g": np.float16}),
    "concat_narrow_partial": _concat([NARROW, NARROW], out_dtypes={"f": np.float16}),
    "concat_many": _concat([MANY, MANY]),
    "concat_pad": _concat([PAD, PAD]),
    "concat_content": _concat([CONTENT, CONTENT]),
    "concat_varint_rows": _concat([VARINT_BAD["rows"], VARINT_BAD["rows"]]),
    "concat_varint_few": _concat([VARINT_BAD["few"], VARINT_BAD["few"]]),
    "concat_varint_range": _concat([VARINT_BAD["range"], VARINT_BAD["range"]]),
    "concat_truncated_first": _concat([TRUNCATED, MIXED]),
    "concat_truncated_second": _concat([MIXED, TRUNCATED]),
    "concat_dtype_disagrees": _concat([FLOATS, build([("scores", F32.astype(np.float64)), ("d", F64)])]),
    "concat_out_numpy": _concat([FLOATS, FLOATS2], out={"scores": ((16, 5), np.float32, False)}),
    "concat_out_device": _concat([FLOATS, FLOATS2], out={"scores": ((16, 5), np.float32, True), "d": ((6,), np.float64, True)}),
    "concat_out_mismatch": _concat([FLOATS, FLOATS2], out={"scores": ((15, 5), np.float32, False)}),
    "concat_out_device_mismatch": _concat([FLOATS, FLOATS2], out={"scores": ((16, 5), np.float64, True)}),
    "concat_out_strings_mismatch": _concat([STRINGS, STRINGS], out={"a": ((3,), np.float32, False)}),
    "padded_floats": _padded([FLOATS, FLOATS2, FLOATS]),
    "padded_floats_device": _padded([FLOATS, FLOATS2, FLOATS], device=True),
    "padded_ragged": _padded([FLOATS, RAGGED, WIDE]),
    "padded_ragged_device": _padded([FLOATS, RAGGED, WIDE], device=True),
    "padded_pad_value": _padded([FLOATS, RAGGED, WIDE], pad_value=-1.5),
    "padded_pad_value_bad": _padded([FLOATS, RAGGED], pad_value="x"),
    "padded_pad_to": _padded([FLOATS, RAGGED, WIDE], pad_to={"scores": (9,)}),
    "padded_pad_to_small": _padded([FLOATS, RAGGED, WIDE], pad_to={"scores": (5,)}),
    "padded_pad_to_rank": _padded([FLOATS, RAGGED], pad_to={"scores": (9, 2)}),
    "padded_mixed": _padded([MIXED, MIXED2]),
    "padded_mixed_device": _padded([MIXED, MIXED2], device=True),
    "padded_mixed_strict": _padded([MIXED, MIXED2], strict=True),
    "padded_keys": _padded([MIXED, MIXED2], keys=["d", "classes"]),
    "padded_varint": _padded([VARINT, VARINT]),
    "padded_strings": _padded([STRINGS, STRINGS]),
    "padded_strings_device": _padded([STRINGS, STRINGS], device=True),
    "padded_half": _padded([HALF, HALF]),
    "padded_half_strict": _padded([HALF, HALF], strict=True),
    "padded_narrow": _padded([NARROW, NARROW], out_dtypes={"f": np.float16, "g": np.float16}),
    "padded_narrow_partial": _padded([NARROW, NARROW], out_dtypes={"f": np.float16}),
    "padded_narrow_strict": _padded([NARROW, NARROW], out_dtypes={"f": np.float16, "g": np.float16}, strict=True),
    "padded_many": _padded([MANY, MANY]),
    "padded_rank0": _padded([RANK0, RANK0]),
    "padded_pad": _padded([PAD, PAD]),
    "padded_content": _padded([CONTENT, CONTENT]),
    "padded_varint_rows": _padded([VARINT_BAD["rows"], VARINT_BAD["rows"]]),
    "padded_varint_few": _padded([VARINT_BAD["few"], VARINT_BAD["few"]]),
    "padded_varint_range": _padded([VARINT_BAD["range"], VARINT_BAD["range"]]),
    "padded_truncated_first": _padded([TRUNCATED, MIXED]),
    "padded_truncated_second": _padded([MIXED, TRUNCATED]),
    "padded_dtype_disagrees": _padded([FLOATS, build([("scores", F32.astype(np.float64)), ("d", F64)])]),
    "padded_out_numpy": _padded([FLOATS, FLOATS2], out={"scores": ((16, 5), np.float32, False)}),
    "padded_out_device": _padded([FLOATS, FLOATS2], out={"scores": ((16, 5), np.float32, True), "d": ((6,), np.float64, True)}),
    "padded_out_unaligned": _padded([FLOATS, FLOATS2], out={"d": ((6,), np.float64, "torch")}),
    "padded_out_mismatch": _padded([FLOATS, FLOATS2], out={"scores": ((15, 5), np.float32, False)}),
    "padded_out_device_mismatch": _padded([FLOATS, FLOATS2], out={"scores": ((16, 5), np.float64, True)}),
    "padded_out_strings_mismatch": _padded([STRINGS, STRINGS], out={"a": ((3,), np.float32, False)}),
    "tensor_protos": lambda c: (c.decode_tensor_protos([SEEDS["t_f32"], SEEDS["t_i32"], SEEDS["t_f64_content"]]), []),
    "tensor_protos_strict": lambda c: (c.decode_tensor_protos([SEEDS["t_f32"], SEEDS["t_i32"], SEEDS["t_f64_content"]], strict=True), []),
    "parse": lambda c: ([sorted(p.keys()) for p in c.parse_predict_responses([FLOATS, MANY, STRINGS])], []),
})


def _kind(a, outs):
    if any(a is o for o in outs):
        return "out"
    root = a
    while isinstance(root.base, np.ndarray):
        root = root.base
    return "view" if root is not a and root.dtype == np.uint8 and a.dtype.kind != "U" else "fresh"


def _summary(v, outs):
    if isinstance(v, DV.DeviceArray):
        host = v.copy_to_host()
        return ["device", host.dtype.str, list(host.shape), hashlib.sha1(host.tobytes()).hexdigest()[:12],
                "out" if any(v is o for o in outs) else "device"]
    if isinstance(v, np.ndarray):
        return ["array", v.dtype.str, list(v.shape), hashlib.sha1(v.tobytes()).hexdigest()[:12], _kind(v, outs)]
    if isinstance(v, DecodedSpec):
        return ["spec", v.name, v.version, v.has_version, v.version_label, v.signature_name]
    if isinstance(v, dict):
        return [[k, _summary(x, outs)] for k, x in v.items()]
    if isinstance(v, (list, tuple)):
        return [_summary(x, outs) for x in v]
    return v


def _outcome(fn):
    try:
        return ["ok", fn()]
    except Exception as e:      # noqa: BLE001 - the exception type is what is pinned
        return ["raise", type(e).__name__]


def _stats(c):
    v = [C.c_uint64() for _ in range(3)]
    N.check(c._lib.b200tfs_decode_stats(c._ctx, *[C.byref(x) for x in v]))
    return [x.value for x in v]


def _call(c, fn, counts):
    counts.clear()
    l0, s0, k0 = c.kernel_launches(), _stats(c), c.concat_device_calls
    outs = []

    def run():
        value, dst = fn(c)
        outs.extend(dst)
        return value
    got = _outcome(run)
    seen = dict(sorted(counts.items()))
    l1, s1, k1 = c.kernel_launches(), _stats(c), c.concat_device_calls
    result = [got[0], _summary(got[1], outs)]
    for a in outs:
        if isinstance(a, DV.DeviceArray):
            a.free()
    return {"result": result, "calls": seen, "launches": l1 - l0, "stats": [b - a for a, b in zip(s0, s1)],
            "concat_device_calls": k1 - k0, "seen_varints": c._seen_varints}


def observe(fn):
    """The four calls of one case, as plain JSON values."""
    lib = N.load()
    counts = {}
    real = {name: getattr(lib, name) for name in COUNTED}

    def counted(name):
        def f(*a):
            counts[name] = counts.get(name, 0) + 1
            return real[name](*a)
        return f
    for name in COUNTED:
        setattr(lib, name, counted(name))
    rec = {}
    try:
        for warm in (False, True):
            c = Codec(0)
            try:
                if warm:
                    c.decode_predict_responses([WARM])
                rec["warm" if warm else "cold"] = [_call(c, fn, counts) for _ in range(2)]
            finally:
                c.close()
    finally:
        for name in COUNTED:
            setattr(lib, name, real[name])
    return json.loads(json.dumps(rec))


@pytest.mark.parametrize("case", sorted(CASES))
def test_route(case):
    assert observe(CASES[case]) == EXPECTED[case]


def test_every_case_has_expectations():
    assert set(CASES) == set(EXPECTED)


EXPECTED = {
    'batch_floats': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['d', ['array', '<f8', [3], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['scores', ['array', '<f4', [8, 5], '8c45f0670cb9', 'view']], ['d', ['array', '<f8', [3], 'f9092f7cccc4', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['d', ['array', '<f8', [3], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [3, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['d', ['array', '<f8', [3], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['scores', ['array', '<f4', [8, 5], '8c45f0670cb9', 'view']], ['d', ['array', '<f8', [3], 'f9092f7cccc4', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['d', ['array', '<f8', [3], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [3, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['d', ['array', '<f8', [3], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['scores', ['array', '<f4', [8, 5], '8c45f0670cb9', 'view']], ['d', ['array', '<f8', [3], 'f9092f7cccc4', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['d', ['array', '<f8', [3], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [3, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['d', ['array', '<f8', [3], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['scores', ['array', '<f4', [8, 5], '8c45f0670cb9', 'view']], ['d', ['array', '<f8', [3], 'f9092f7cccc4', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['d', ['array', '<f8', [3], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [3, 0, 0]},
        ],
    },
    'batch_mixed': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 10, 'result': ['ok', [[[['ids', ['array', '<i8', [3, 7], '52cb4304056a', 'fresh']], ['mask', ['array', '|b1', [9], '4f8cb9968539', 'fresh']], ['small', ['array', '<i4', [5], '430c389090db', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['d', ['array', '<f8', [3, 1], '7f0639ce5dac', 'view']], ['classes', ['array', '<i8', [8, 5], '431851990268', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['a', ['array', '<f4', [4], '8f6809c988e5', 'view']], ['s', ['array', '<U3', [2], '1424e0e98d55', 'fresh']], ['ids', ['array', '<i8', [6], '2b33b5254d22', 'fresh']], ['m', ['array', '|b1', [5], '78385b49bf10', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['f', ['array', '<f4', [5], '10f358f16a8b', 'view']], ['h', ['array', '<f2', [6], '8a8ce3354514', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 3]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['ids', ['array', '<i8', [3, 7], '52cb4304056a', 'view']], ['mask', ['array', '|b1', [9], '4f8cb9968539', 'view']], ['small', ['array', '<i4', [5], '430c389090db', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['classes', ['array', '<i8', [8, 5], '431851990268', 'view']], ['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['d', ['array', '<f8', [3, 1], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['a', ['array', '<f4', [4], '8f6809c988e5', 'view']], ['ids', ['array', '<i8', [6], '2b33b5254d22', 'view']], ['m', ['array', '|b1', [5], '78385b49bf10', 'view']], ['s', ['array', '<U3', [2], '1424e0e98d55', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['h', ['array', '<f2', [6], '8a8ce3354514', 'view']], ['f', ['array', '<f4', [5], '10f358f16a8b', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 3]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['ids', ['array', '<i8', [3, 7], '52cb4304056a', 'view']], ['mask', ['array', '|b1', [9], '4f8cb9968539', 'view']], ['small', ['array', '<i4', [5], '430c389090db', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['classes', ['array', '<i8', [8, 5], '431851990268', 'view']], ['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['d', ['array', '<f8', [3, 1], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['a', ['array', '<f4', [4], '8f6809c988e5', 'view']], ['ids', ['array', '<i8', [6], '2b33b5254d22', 'view']], ['m', ['array', '|b1', [5], '78385b49bf10', 'view']], ['s', ['array', '<U3', [2], '1424e0e98d55', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['h', ['array', '<f2', [6], '8a8ce3354514', 'view']], ['f', ['array', '<f4', [5], '10f358f16a8b', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 3]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['ids', ['array', '<i8', [3, 7], '52cb4304056a', 'view']], ['mask', ['array', '|b1', [9], '4f8cb9968539', 'view']], ['small', ['array', '<i4', [5], '430c389090db', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['classes', ['array', '<i8', [8, 5], '431851990268', 'view']], ['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['d', ['array', '<f8', [3, 1], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['a', ['array', '<f4', [4], '8f6809c988e5', 'view']], ['ids', ['array', '<i8', [6], '2b33b5254d22', 'view']], ['m', ['array', '|b1', [5], '78385b49bf10', 'view']], ['s', ['array', '<U3', [2], '1424e0e98d55', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['h', ['array', '<f2', [6], '8a8ce3354514', 'view']], ['f', ['array', '<f4', [5], '10f358f16a8b', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 3]},
        ],
    },
    'batch_mixed_strict': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 3, 'result': ['ok', [[[['ids', ['array', '<i8', [3, 7], '52cb4304056a', 'fresh']], ['mask', ['array', '|b1', [9], '4f8cb9968539', 'fresh']], ['small', ['array', '<i4', [5], '430c389090db', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['d', ['array', '<f8', [3, 1], '7f0639ce5dac', 'view']], ['classes', ['array', '<i8', [8, 5], '431851990268', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['a', ['array', '<f4', [4], '8f6809c988e5', 'view']], ['s', ['array', '<U3', [2], '1424e0e98d55', 'fresh']], ['ids', ['array', '<i8', [6], '2b33b5254d22', 'fresh']], ['m', ['array', '|b1', [5], '78385b49bf10', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['f', ['array', '<f4', [5], '10f358f16a8b', 'view']], ['h', ['array', '<f2', [6], 'a0bfed79c547', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 3]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[[['ids', ['array', '<i8', [3, 7], '52cb4304056a', 'view']], ['mask', ['array', '|b1', [9], '4f8cb9968539', 'view']], ['small', ['array', '<i4', [5], '430c389090db', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['classes', ['array', '<i8', [8, 5], '431851990268', 'view']], ['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['d', ['array', '<f8', [3, 1], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['a', ['array', '<f4', [4], '8f6809c988e5', 'view']], ['ids', ['array', '<i8', [6], '2b33b5254d22', 'view']], ['m', ['array', '|b1', [5], '78385b49bf10', 'view']], ['s', ['array', '<U3', [2], '1424e0e98d55', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['f', ['array', '<f4', [5], '10f358f16a8b', 'view']], ['h', ['array', '<f2', [6], 'a0bfed79c547', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 3]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[[['ids', ['array', '<i8', [3, 7], '52cb4304056a', 'view']], ['mask', ['array', '|b1', [9], '4f8cb9968539', 'view']], ['small', ['array', '<i4', [5], '430c389090db', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['classes', ['array', '<i8', [8, 5], '431851990268', 'view']], ['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['d', ['array', '<f8', [3, 1], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['a', ['array', '<f4', [4], '8f6809c988e5', 'view']], ['ids', ['array', '<i8', [6], '2b33b5254d22', 'view']], ['m', ['array', '|b1', [5], '78385b49bf10', 'view']], ['s', ['array', '<U3', [2], '1424e0e98d55', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['f', ['array', '<f4', [5], '10f358f16a8b', 'view']], ['h', ['array', '<f2', [6], 'a0bfed79c547', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 3]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[[['ids', ['array', '<i8', [3, 7], '52cb4304056a', 'view']], ['mask', ['array', '|b1', [9], '4f8cb9968539', 'view']], ['small', ['array', '<i4', [5], '430c389090db', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['classes', ['array', '<i8', [8, 5], '431851990268', 'view']], ['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['d', ['array', '<f8', [3, 1], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['a', ['array', '<f4', [4], '8f6809c988e5', 'view']], ['ids', ['array', '<i8', [6], '2b33b5254d22', 'view']], ['m', ['array', '|b1', [5], '78385b49bf10', 'view']], ['s', ['array', '<U3', [2], '1424e0e98d55', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['f', ['array', '<f4', [5], '10f358f16a8b', 'view']], ['h', ['array', '<f2', [6], 'a0bfed79c547', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 3]},
        ],
    },
    'batch_with_malformed': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_parse_responses_host': 1}, 'concat_device_calls': 0, 'launches': 2, 'result': ['raise', 'DecodeError'], 'seen_varints': False, 'stats': [1, 0, 1]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_parse_responses_host': 1}, 'concat_device_calls': 0, 'launches': 2, 'result': ['raise', 'DecodeError'], 'seen_varints': False, 'stats': [1, 0, 1]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_parse_responses_host': 1}, 'concat_device_calls': 0, 'launches': 2, 'result': ['raise', 'DecodeError'], 'seen_varints': True, 'stats': [1, 0, 1]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_parse_responses_host': 1}, 'concat_device_calls': 0, 'launches': 2, 'result': ['raise', 'DecodeError'], 'seen_varints': True, 'stats': [1, 0, 1]},
        ],
    },
    'batch_with_many': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_parse_responses_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 3, 'result': ['ok', [[[['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'fresh']], ['d', ['array', '<f8', [3], '7f0639ce5dac', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['o0', ['array', '<f4', [5], '10f358f16a8b', 'fresh']], ['o1', ['array', '<f4', [5], 'df5a3f2b035e', 'fresh']], ['o2', ['array', '<f4', [5], '8f264031c27f', 'fresh']], ['o3', ['array', '<f4', [5], 'd52326878a3d', 'fresh']], ['o4', ['array', '<f4', [5], '9d03c78062f2', 'fresh']], ['o5', ['array', '<f4', [5], '5d3443a4d60e', 'fresh']], ['o6', ['array', '<f4', [5], '7caf92caf1a5', 'fresh']], ['o7', ['array', '<f4', [5], 'b1108aae2c65', 'fresh']], ['o8', ['array', '<f4', [5], '8215e6f03231', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [1, 0, 1]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_parse_responses_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 3, 'result': ['ok', [[[['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'fresh']], ['d', ['array', '<f8', [3], '7f0639ce5dac', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['o0', ['array', '<f4', [5], '10f358f16a8b', 'fresh']], ['o1', ['array', '<f4', [5], 'df5a3f2b035e', 'fresh']], ['o2', ['array', '<f4', [5], '8f264031c27f', 'fresh']], ['o3', ['array', '<f4', [5], 'd52326878a3d', 'fresh']], ['o4', ['array', '<f4', [5], '9d03c78062f2', 'fresh']], ['o5', ['array', '<f4', [5], '5d3443a4d60e', 'fresh']], ['o6', ['array', '<f4', [5], '7caf92caf1a5', 'fresh']], ['o7', ['array', '<f4', [5], 'b1108aae2c65', 'fresh']], ['o8', ['array', '<f4', [5], '8215e6f03231', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [1, 0, 1]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_parse_responses_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 3, 'result': ['ok', [[[['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'fresh']], ['d', ['array', '<f8', [3], '7f0639ce5dac', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['o0', ['array', '<f4', [5], '10f358f16a8b', 'fresh']], ['o1', ['array', '<f4', [5], 'df5a3f2b035e', 'fresh']], ['o2', ['array', '<f4', [5], '8f264031c27f', 'fresh']], ['o3', ['array', '<f4', [5], 'd52326878a3d', 'fresh']], ['o4', ['array', '<f4', [5], '9d03c78062f2', 'fresh']], ['o5', ['array', '<f4', [5], '5d3443a4d60e', 'fresh']], ['o6', ['array', '<f4', [5], '7caf92caf1a5', 'fresh']], ['o7', ['array', '<f4', [5], 'b1108aae2c65', 'fresh']], ['o8', ['array', '<f4', [5], '8215e6f03231', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 1]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_parse_responses_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 3, 'result': ['ok', [[[['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'fresh']], ['d', ['array', '<f8', [3], '7f0639ce5dac', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['o0', ['array', '<f4', [5], '10f358f16a8b', 'fresh']], ['o1', ['array', '<f4', [5], 'df5a3f2b035e', 'fresh']], ['o2', ['array', '<f4', [5], '8f264031c27f', 'fresh']], ['o3', ['array', '<f4', [5], 'd52326878a3d', 'fresh']], ['o4', ['array', '<f4', [5], '9d03c78062f2', 'fresh']], ['o5', ['array', '<f4', [5], '5d3443a4d60e', 'fresh']], ['o6', ['array', '<f4', [5], '7caf92caf1a5', 'fresh']], ['o7', ['array', '<f4', [5], 'b1108aae2c65', 'fresh']], ['o8', ['array', '<f4', [5], '8215e6f03231', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 1]},
        ],
    },
    'cast_f64': {
        'cold': [
            {'calls': {'b200tfs_parse_responses_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_parse_responses_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_parse_responses_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_parse_responses_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'cast_ids': {
        'cold': [
            {'calls': {'b200tfs_parse_responses_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_parse_responses_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_parse_responses_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_parse_responses_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'concat_content': {
        'cold': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[['c', ['array', '<f4', [16, 5], '0faa8a48c67b', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[['c', ['array', '<f4', [16, 5], '0faa8a48c67b', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[['c', ['array', '<f4', [16, 5], '0faa8a48c67b', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[['c', ['array', '<f4', [16, 5], '0faa8a48c67b', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'concat_dtype_disagrees': {
        'cold': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'concat_floats': {
        'cold': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['scores', ['array', '<f4', [24, 5], '907117f39572', 'fresh']], ['d', ['array', '<f8', [9], 'ac70ecbf4f0c', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['scores', ['array', '<f4', [24, 5], '907117f39572', 'fresh']], ['d', ['array', '<f8', [9], 'ac70ecbf4f0c', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['scores', ['array', '<f4', [24, 5], '907117f39572', 'fresh']], ['d', ['array', '<f8', [9], 'ac70ecbf4f0c', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['scores', ['array', '<f4', [24, 5], '907117f39572', 'fresh']], ['d', ['array', '<f8', [9], 'ac70ecbf4f0c', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'concat_floats_device': {
        'cold': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['scores', ['device', '<f4', [24, 5], '907117f39572', 'device']], ['d', ['device', '<f8', [9], 'ac70ecbf4f0c', 'device']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['scores', ['device', '<f4', [24, 5], '907117f39572', 'device']], ['d', ['device', '<f8', [9], 'ac70ecbf4f0c', 'device']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['scores', ['device', '<f4', [24, 5], '907117f39572', 'device']], ['d', ['device', '<f8', [9], 'ac70ecbf4f0c', 'device']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['scores', ['device', '<f4', [24, 5], '907117f39572', 'device']], ['d', ['device', '<f8', [9], 'ac70ecbf4f0c', 'device']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'concat_half': {
        'cold': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['h', ['array', '<f2', [12], 'd7d38c467a05', 'fresh']], ['f', ['array', '<f4', [10], '978ac77ea8bf', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['h', ['array', '<f2', [12], 'd7d38c467a05', 'fresh']], ['f', ['array', '<f4', [10], '978ac77ea8bf', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['h', ['array', '<f2', [12], 'd7d38c467a05', 'fresh']], ['f', ['array', '<f4', [10], '978ac77ea8bf', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['h', ['array', '<f2', [12], 'd7d38c467a05', 'fresh']], ['f', ['array', '<f4', [10], '978ac77ea8bf', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'concat_half_strict': {
        'cold': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs': 1}, 'concat_device_calls': 1, 'launches': 8, 'result': ['ok', [[['h', ['array', '<f2', [12], 'a612ac46cb97', 'fresh']], ['f', ['array', '<f4', [10], '978ac77ea8bf', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs': 1}, 'concat_device_calls': 1, 'launches': 8, 'result': ['ok', [[['h', ['array', '<f2', [12], 'a612ac46cb97', 'fresh']], ['f', ['array', '<f4', [10], '978ac77ea8bf', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs': 1}, 'concat_device_calls': 1, 'launches': 8, 'result': ['ok', [[['h', ['array', '<f2', [12], 'a612ac46cb97', 'fresh']], ['f', ['array', '<f4', [10], '978ac77ea8bf', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs': 1}, 'concat_device_calls': 1, 'launches': 8, 'result': ['ok', [[['h', ['array', '<f2', [12], 'a612ac46cb97', 'fresh']], ['f', ['array', '<f4', [10], '978ac77ea8bf', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'concat_keys': {
        'cold': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['d', ['array', '<f8', [4, 1], '29fc26da5c1c', 'fresh']], ['classes', ['array', '<i8', [10, 5], 'db935af57046', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['d', ['array', '<f8', [4, 1], '29fc26da5c1c', 'fresh']], ['classes', ['array', '<i8', [10, 5], 'db935af57046', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['d', ['array', '<f8', [4, 1], '29fc26da5c1c', 'fresh']], ['classes', ['array', '<i8', [10, 5], 'db935af57046', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['d', ['array', '<f8', [4, 1], '29fc26da5c1c', 'fresh']], ['classes', ['array', '<i8', [10, 5], 'db935af57046', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'concat_many': {
        'cold': [
            {'calls': {'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[['o0', ['array', '<f4', [10], '978ac77ea8bf', 'fresh']], ['o1', ['array', '<f4', [10], '9bd4809dc080', 'fresh']], ['o2', ['array', '<f4', [10], '603b11843256', 'fresh']], ['o3', ['array', '<f4', [10], '12388578a29e', 'fresh']], ['o4', ['array', '<f4', [10], '50493d3f1088', 'fresh']], ['o5', ['array', '<f4', [10], '159f97f92d1a', 'fresh']], ['o6', ['array', '<f4', [10], '4d18a2bb7161', 'fresh']], ['o7', ['array', '<f4', [10], '361fa970ef6e', 'fresh']], ['o8', ['array', '<f4', [10], '2b195ee6133a', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[['o0', ['array', '<f4', [10], '978ac77ea8bf', 'fresh']], ['o1', ['array', '<f4', [10], '9bd4809dc080', 'fresh']], ['o2', ['array', '<f4', [10], '603b11843256', 'fresh']], ['o3', ['array', '<f4', [10], '12388578a29e', 'fresh']], ['o4', ['array', '<f4', [10], '50493d3f1088', 'fresh']], ['o5', ['array', '<f4', [10], '159f97f92d1a', 'fresh']], ['o6', ['array', '<f4', [10], '4d18a2bb7161', 'fresh']], ['o7', ['array', '<f4', [10], '361fa970ef6e', 'fresh']], ['o8', ['array', '<f4', [10], '2b195ee6133a', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[['o0', ['array', '<f4', [10], '978ac77ea8bf', 'fresh']], ['o1', ['array', '<f4', [10], '9bd4809dc080', 'fresh']], ['o2', ['array', '<f4', [10], '603b11843256', 'fresh']], ['o3', ['array', '<f4', [10], '12388578a29e', 'fresh']], ['o4', ['array', '<f4', [10], '50493d3f1088', 'fresh']], ['o5', ['array', '<f4', [10], '159f97f92d1a', 'fresh']], ['o6', ['array', '<f4', [10], '4d18a2bb7161', 'fresh']], ['o7', ['array', '<f4', [10], '361fa970ef6e', 'fresh']], ['o8', ['array', '<f4', [10], '2b195ee6133a', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[['o0', ['array', '<f4', [10], '978ac77ea8bf', 'fresh']], ['o1', ['array', '<f4', [10], '9bd4809dc080', 'fresh']], ['o2', ['array', '<f4', [10], '603b11843256', 'fresh']], ['o3', ['array', '<f4', [10], '12388578a29e', 'fresh']], ['o4', ['array', '<f4', [10], '50493d3f1088', 'fresh']], ['o5', ['array', '<f4', [10], '159f97f92d1a', 'fresh']], ['o6', ['array', '<f4', [10], '4d18a2bb7161', 'fresh']], ['o7', ['array', '<f4', [10], '361fa970ef6e', 'fresh']], ['o8', ['array', '<f4', [10], '2b195ee6133a', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'concat_mixed': {
        'cold': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_d2h': 3, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['classes', ['array', '<i8', [10, 5], 'db935af57046', 'fresh']], ['scores', ['array', '<f4', [10, 5], '61c2992f9901', 'fresh']], ['d', ['array', '<f8', [4, 1], '29fc26da5c1c', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_d2h': 3, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['classes', ['array', '<i8', [10, 5], 'db935af57046', 'fresh']], ['scores', ['array', '<f4', [10, 5], '61c2992f9901', 'fresh']], ['d', ['array', '<f8', [4, 1], '29fc26da5c1c', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_d2h': 3, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['classes', ['array', '<i8', [10, 5], 'db935af57046', 'fresh']], ['scores', ['array', '<f4', [10, 5], '61c2992f9901', 'fresh']], ['d', ['array', '<f8', [4, 1], '29fc26da5c1c', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_d2h': 3, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['classes', ['array', '<i8', [10, 5], 'db935af57046', 'fresh']], ['scores', ['array', '<f4', [10, 5], '61c2992f9901', 'fresh']], ['d', ['array', '<f8', [4, 1], '29fc26da5c1c', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'concat_mixed_device': {
        'cold': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['classes', ['device', '<i8', [10, 5], 'db935af57046', 'device']], ['scores', ['device', '<f4', [10, 5], '61c2992f9901', 'device']], ['d', ['device', '<f8', [4, 1], '29fc26da5c1c', 'device']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['classes', ['device', '<i8', [10, 5], 'db935af57046', 'device']], ['scores', ['device', '<f4', [10, 5], '61c2992f9901', 'device']], ['d', ['device', '<f8', [4, 1], '29fc26da5c1c', 'device']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['classes', ['device', '<i8', [10, 5], 'db935af57046', 'device']], ['scores', ['device', '<f4', [10, 5], '61c2992f9901', 'device']], ['d', ['device', '<f8', [4, 1], '29fc26da5c1c', 'device']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['classes', ['device', '<i8', [10, 5], 'db935af57046', 'device']], ['scores', ['device', '<f4', [10, 5], '61c2992f9901', 'device']], ['d', ['device', '<f8', [4, 1], '29fc26da5c1c', 'device']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'concat_mixed_strict': {
        'cold': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_d2h': 3, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['classes', ['array', '<i8', [10, 5], 'db935af57046', 'fresh']], ['scores', ['array', '<f4', [10, 5], '61c2992f9901', 'fresh']], ['d', ['array', '<f8', [4, 1], '29fc26da5c1c', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_d2h': 3, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['classes', ['array', '<i8', [10, 5], 'db935af57046', 'fresh']], ['scores', ['array', '<f4', [10, 5], '61c2992f9901', 'fresh']], ['d', ['array', '<f8', [4, 1], '29fc26da5c1c', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_d2h': 3, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['classes', ['array', '<i8', [10, 5], 'db935af57046', 'fresh']], ['scores', ['array', '<f4', [10, 5], '61c2992f9901', 'fresh']], ['d', ['array', '<f8', [4, 1], '29fc26da5c1c', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_d2h': 3, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['classes', ['array', '<i8', [10, 5], 'db935af57046', 'fresh']], ['scores', ['array', '<f4', [10, 5], '61c2992f9901', 'fresh']], ['d', ['array', '<f8', [4, 1], '29fc26da5c1c', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'concat_narrow': {
        'cold': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_d2h': 3, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1, 'b200tfs_set_decode_cast': 2}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['f', ['array', '<f2', [60, 7], '1ef8d77aafaa', 'fresh']], ['g', ['array', '<f2', [198], '01c90ef1748f', 'fresh']], ['ids', ['array', '<i8', [100], '4b0fdc7daed0', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_d2h': 3, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1, 'b200tfs_set_decode_cast': 2}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['f', ['array', '<f2', [60, 7], '1ef8d77aafaa', 'fresh']], ['g', ['array', '<f2', [198], '01c90ef1748f', 'fresh']], ['ids', ['array', '<i8', [100], '4b0fdc7daed0', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_d2h': 3, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1, 'b200tfs_set_decode_cast': 2}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['f', ['array', '<f2', [60, 7], '1ef8d77aafaa', 'fresh']], ['g', ['array', '<f2', [198], '01c90ef1748f', 'fresh']], ['ids', ['array', '<i8', [100], '4b0fdc7daed0', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_d2h': 3, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1, 'b200tfs_set_decode_cast': 2}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['f', ['array', '<f2', [60, 7], '1ef8d77aafaa', 'fresh']], ['g', ['array', '<f2', [198], '01c90ef1748f', 'fresh']], ['ids', ['array', '<i8', [100], '4b0fdc7daed0', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'concat_narrow_partial': {
        'cold': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 10, 'result': ['ok', [[['f', ['array', '<f2', [60, 7], '1ef8d77aafaa', 'fresh']], ['g', ['array', '<f4', [198], 'ea065140f6b0', 'fresh']], ['ids', ['array', '<i8', [100], '4b0fdc7daed0', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 10, 'result': ['ok', [[['f', ['array', '<f2', [60, 7], '1ef8d77aafaa', 'fresh']], ['g', ['array', '<f4', [198], 'ea065140f6b0', 'fresh']], ['ids', ['array', '<i8', [100], '4b0fdc7daed0', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 10, 'result': ['ok', [[['f', ['array', '<f2', [60, 7], '1ef8d77aafaa', 'fresh']], ['g', ['array', '<f4', [198], 'ea065140f6b0', 'fresh']], ['ids', ['array', '<i8', [100], '4b0fdc7daed0', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 10, 'result': ['ok', [[['f', ['array', '<f2', [60, 7], '1ef8d77aafaa', 'fresh']], ['g', ['array', '<f4', [198], 'ea065140f6b0', 'fresh']], ['ids', ['array', '<i8', [100], '4b0fdc7daed0', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'concat_out_device': {
        'cold': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_h2d': 3, 'b200tfs_response_keys': 1}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['scores', ['device', '<f4', [16, 5], '9808d3628a01', 'out']], ['d', ['device', '<f8', [6], '9f573d120c9b', 'out']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_h2d': 3, 'b200tfs_response_keys': 1}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['scores', ['device', '<f4', [16, 5], '9808d3628a01', 'out']], ['d', ['device', '<f8', [6], '9f573d120c9b', 'out']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_h2d': 3, 'b200tfs_response_keys': 1}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['scores', ['device', '<f4', [16, 5], '9808d3628a01', 'out']], ['d', ['device', '<f8', [6], '9f573d120c9b', 'out']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_h2d': 3, 'b200tfs_response_keys': 1}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['scores', ['device', '<f4', [16, 5], '9808d3628a01', 'out']], ['d', ['device', '<f8', [6], '9f573d120c9b', 'out']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'concat_out_device_mismatch': {
        'cold': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 0, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 0, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 0, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 0, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'concat_out_mismatch': {
        'cold': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 0, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 0, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 0, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 0, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'concat_out_numpy': {
        'cold': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['scores', ['array', '<f4', [16, 5], '9808d3628a01', 'out']], ['d', ['array', '<f8', [6], '9f573d120c9b', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['scores', ['array', '<f4', [16, 5], '9808d3628a01', 'out']], ['d', ['array', '<f8', [6], '9f573d120c9b', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['scores', ['array', '<f4', [16, 5], '9808d3628a01', 'out']], ['d', ['array', '<f8', [6], '9f573d120c9b', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 1, 'launches': 6, 'result': ['ok', [[['scores', ['array', '<f4', [16, 5], '9808d3628a01', 'out']], ['d', ['array', '<f8', [6], '9f573d120c9b', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'concat_out_strings_mismatch': {
        'cold': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 12, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 12, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 12, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 12, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'concat_pad': {
        'cold': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['p', ['array', '<f4', [12], 'bb69489226a6', 'fresh']], ['z', ['array', '<f4', [8], 'de8a847bff8c', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['p', ['array', '<f4', [12], 'bb69489226a6', 'fresh']], ['z', ['array', '<f4', [8], 'de8a847bff8c', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['p', ['array', '<f4', [12], 'bb69489226a6', 'fresh']], ['z', ['array', '<f4', [8], 'de8a847bff8c', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['p', ['array', '<f4', [12], 'bb69489226a6', 'fresh']], ['z', ['array', '<f4', [8], 'de8a847bff8c', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'concat_strings': {
        'cold': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 12, 'result': ['ok', [[['a', ['array', '<f4', [8], '7e0c4ddcde8e', 'fresh']], ['ids', ['array', '<i8', [12], 'b1e1d436fa4c', 'fresh']], ['m', ['array', '|b1', [10], '86cd1efe8a37', 'fresh']], ['s', ['array', '<U3', [4], '45a441b904fa', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 12, 'result': ['ok', [[['a', ['array', '<f4', [8], '7e0c4ddcde8e', 'fresh']], ['ids', ['array', '<i8', [12], 'b1e1d436fa4c', 'fresh']], ['m', ['array', '|b1', [10], '86cd1efe8a37', 'fresh']], ['s', ['array', '<U3', [4], '45a441b904fa', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 12, 'result': ['ok', [[['a', ['array', '<f4', [8], '7e0c4ddcde8e', 'fresh']], ['ids', ['array', '<i8', [12], 'b1e1d436fa4c', 'fresh']], ['m', ['array', '|b1', [10], '86cd1efe8a37', 'fresh']], ['s', ['array', '<U3', [4], '45a441b904fa', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 12, 'result': ['ok', [[['a', ['array', '<f4', [8], '7e0c4ddcde8e', 'fresh']], ['ids', ['array', '<i8', [12], 'b1e1d436fa4c', 'fresh']], ['m', ['array', '|b1', [10], '86cd1efe8a37', 'fresh']], ['s', ['array', '<U3', [4], '45a441b904fa', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'concat_strings_device': {
        'cold': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_memcpy_h2d': 3, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 12, 'result': ['raise', 'TypeError'], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_memcpy_h2d': 3, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 12, 'result': ['raise', 'TypeError'], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_memcpy_h2d': 3, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 12, 'result': ['raise', 'TypeError'], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_memcpy_h2d': 3, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 12, 'result': ['raise', 'TypeError'], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'concat_truncated_first': {
        'cold': [
            {'calls': {'b200tfs_parse_responses_host': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'DecodeError'], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_parse_responses_host': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'DecodeError'], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_parse_responses_host': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'DecodeError'], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_parse_responses_host': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'DecodeError'], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'concat_truncated_second': {
        'cold': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['raise', 'DecodeError'], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['raise', 'DecodeError'], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['raise', 'DecodeError'], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['raise', 'DecodeError'], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'concat_varint_few': {
        'cold': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 8, 'result': ['ok', [[['x', ['array', '<i8', [8], 'd1b4082d226e', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 8, 'result': ['ok', [[['x', ['array', '<i8', [8], 'd1b4082d226e', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 8, 'result': ['ok', [[['x', ['array', '<i8', [8], 'd1b4082d226e', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 8, 'result': ['ok', [[['x', ['array', '<i8', [8], 'd1b4082d226e', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'concat_varint_range': {
        'cold': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_parse_responses_host': 1, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 14, 'result': ['raise', 'OverflowError'], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_parse_responses_host': 1, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 14, 'result': ['raise', 'OverflowError'], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_parse_responses_host': 1, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 14, 'result': ['raise', 'OverflowError'], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_parse_responses_host': 1, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 14, 'result': ['raise', 'OverflowError'], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'concat_varint_rows': {
        'cold': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_d2h': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs': 1}, 'concat_device_calls': 1, 'launches': 11, 'result': ['ok', [[['x', ['array', '<i4', [6], 'bc820beafeab', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_d2h': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs': 1}, 'concat_device_calls': 1, 'launches': 11, 'result': ['ok', [[['x', ['array', '<i4', [6], 'bc820beafeab', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_d2h': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs': 1}, 'concat_device_calls': 1, 'launches': 11, 'result': ['ok', [[['x', ['array', '<i4', [6], 'bc820beafeab', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_concat_layout': 1, 'b200tfs_concat_results': 1, 'b200tfs_decode_concat': 1, 'b200tfs_memcpy_d2h': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs': 1}, 'concat_device_calls': 1, 'launches': 11, 'result': ['ok', [[['x', ['array', '<i4', [6], 'bc820beafeab', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'decode_bf16_strict': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'KeyError'], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['raise', 'KeyError'], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['raise', 'KeyError'], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['raise', 'KeyError'], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_bf16_tolerant': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['b', ['array', '<V2', [2], '18d36867d977', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['b', ['array', '<V2', [2], '18d36867d977', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['b', ['array', '<V2', [2], '18d36867d977', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['b', ['array', '<V2', [2], '18d36867d977', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_complex_strict': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_complex_tolerant': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['c', ['array', '<c8', [2], '30c3c8e10060', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['c', ['array', '<c8', [2], '30c3c8e10060', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['c', ['array', '<c8', [2], '30c3c8e10060', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['c', ['array', '<c8', [2], '30c3c8e10060', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_content_strict': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_content_tolerant': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 2, 'result': ['ok', [[[['c', ['array', '<f4', [8, 5], '640ba4d3c6af', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 2, 'result': ['ok', [[[['c', ['array', '<f4', [8, 5], '640ba4d3c6af', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 2, 'result': ['ok', [[[['c', ['array', '<f4', [8, 5], '640ba4d3c6af', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 2, 'result': ['ok', [[[['c', ['array', '<f4', [8, 5], '640ba4d3c6af', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_empty_strict': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[], ['spec', '', 0, False, '', '']]]], 'seen_varints': False, 'stats': [0, 0, 1]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[], ['spec', '', 0, False, '', '']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[], ['spec', '', 0, False, '', '']]]], 'seen_varints': True, 'stats': [0, 0, 1]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[], ['spec', '', 0, False, '', '']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_empty_tolerant': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[], ['spec', '', 0, False, '', '']]]], 'seen_varints': False, 'stats': [0, 0, 1]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[], ['spec', '', 0, False, '', '']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[], ['spec', '', 0, False, '', '']]]], 'seen_varints': True, 'stats': [0, 0, 1]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[], ['spec', '', 0, False, '', '']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_flipped_strict': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['d', ['array', '<f8', [3], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['d', ['array', '<f8', [3], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['d', ['array', '<f8', [3], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['d', ['array', '<f8', [3], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_flipped_tolerant': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['d', ['array', '<f8', [3], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['d', ['array', '<f8', [3], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['d', ['array', '<f8', [3], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['d', ['array', '<f8', [3], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_floats_strict': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['d', ['array', '<f8', [3], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['d', ['array', '<f8', [3], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['d', ['array', '<f8', [3], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['d', ['array', '<f8', [3], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_floats_tolerant': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['d', ['array', '<f8', [3], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['d', ['array', '<f8', [3], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['d', ['array', '<f8', [3], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['d', ['array', '<f8', [3], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_half_strict': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 3, 'result': ['ok', [[[['f', ['array', '<f4', [5], '10f358f16a8b', 'view']], ['h', ['array', '<f2', [6], 'a0bfed79c547', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[[['f', ['array', '<f4', [5], '10f358f16a8b', 'view']], ['h', ['array', '<f2', [6], 'a0bfed79c547', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[[['f', ['array', '<f4', [5], '10f358f16a8b', 'view']], ['h', ['array', '<f2', [6], 'a0bfed79c547', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[[['f', ['array', '<f4', [5], '10f358f16a8b', 'view']], ['h', ['array', '<f2', [6], 'a0bfed79c547', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_half_tolerant': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['f', ['array', '<f4', [5], '10f358f16a8b', 'view']], ['h', ['array', '<f2', [6], '8a8ce3354514', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['h', ['array', '<f2', [6], '8a8ce3354514', 'view']], ['f', ['array', '<f4', [5], '10f358f16a8b', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['h', ['array', '<f2', [6], '8a8ce3354514', 'view']], ['f', ['array', '<f4', [5], '10f358f16a8b', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['h', ['array', '<f2', [6], '8a8ce3354514', 'view']], ['f', ['array', '<f4', [5], '10f358f16a8b', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_many_mixed_strict': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_parse_responses_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 5, 'result': ['ok', [[[['o0', ['array', '<i8', [7], '6984488c7681', 'fresh']], ['o1', ['array', '<f4', [5], '417230de77a6', 'fresh']], ['o2', ['array', '<i8', [7], '47f0a2d7b99f', 'fresh']], ['o3', ['array', '<f4', [5], 'c00c6de9a76d', 'fresh']], ['o4', ['array', '<i8', [7], '607bc080dbb9', 'fresh']], ['o5', ['array', '<f4', [5], '51fb7d8c9563', 'fresh']], ['o6', ['array', '<i8', [7], '6984488c7681', 'fresh']], ['o7', ['array', '<f4', [5], '0310ddc723fc', 'fresh']], ['o8', ['array', '<i8', [7], '47f0a2d7b99f', 'fresh']], ['o9', ['array', '<f4', [5], '417230de77a6', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 1]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_parse_responses_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 5, 'result': ['ok', [[[['o0', ['array', '<i8', [7], '6984488c7681', 'fresh']], ['o1', ['array', '<f4', [5], '417230de77a6', 'fresh']], ['o2', ['array', '<i8', [7], '47f0a2d7b99f', 'fresh']], ['o3', ['array', '<f4', [5], 'c00c6de9a76d', 'fresh']], ['o4', ['array', '<i8', [7], '607bc080dbb9', 'fresh']], ['o5', ['array', '<f4', [5], '51fb7d8c9563', 'fresh']], ['o6', ['array', '<i8', [7], '6984488c7681', 'fresh']], ['o7', ['array', '<f4', [5], '0310ddc723fc', 'fresh']], ['o8', ['array', '<i8', [7], '47f0a2d7b99f', 'fresh']], ['o9', ['array', '<f4', [5], '417230de77a6', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 1]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_parse_responses_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 5, 'result': ['ok', [[[['o0', ['array', '<i8', [7], '6984488c7681', 'fresh']], ['o1', ['array', '<f4', [5], '417230de77a6', 'fresh']], ['o2', ['array', '<i8', [7], '47f0a2d7b99f', 'fresh']], ['o3', ['array', '<f4', [5], 'c00c6de9a76d', 'fresh']], ['o4', ['array', '<i8', [7], '607bc080dbb9', 'fresh']], ['o5', ['array', '<f4', [5], '51fb7d8c9563', 'fresh']], ['o6', ['array', '<i8', [7], '6984488c7681', 'fresh']], ['o7', ['array', '<f4', [5], '0310ddc723fc', 'fresh']], ['o8', ['array', '<i8', [7], '47f0a2d7b99f', 'fresh']], ['o9', ['array', '<f4', [5], '417230de77a6', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 1]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_parse_responses_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 5, 'result': ['ok', [[[['o0', ['array', '<i8', [7], '6984488c7681', 'fresh']], ['o1', ['array', '<f4', [5], '417230de77a6', 'fresh']], ['o2', ['array', '<i8', [7], '47f0a2d7b99f', 'fresh']], ['o3', ['array', '<f4', [5], 'c00c6de9a76d', 'fresh']], ['o4', ['array', '<i8', [7], '607bc080dbb9', 'fresh']], ['o5', ['array', '<f4', [5], '51fb7d8c9563', 'fresh']], ['o6', ['array', '<i8', [7], '6984488c7681', 'fresh']], ['o7', ['array', '<f4', [5], '0310ddc723fc', 'fresh']], ['o8', ['array', '<i8', [7], '47f0a2d7b99f', 'fresh']], ['o9', ['array', '<f4', [5], '417230de77a6', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 1]},
        ],
    },
    'decode_many_mixed_tolerant': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_parse_responses_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 10, 'result': ['ok', [[[['o0', ['array', '<i8', [7], '6984488c7681', 'fresh']], ['o1', ['array', '<f4', [5], '417230de77a6', 'fresh']], ['o2', ['array', '<i8', [7], '47f0a2d7b99f', 'fresh']], ['o3', ['array', '<f4', [5], 'c00c6de9a76d', 'fresh']], ['o4', ['array', '<i8', [7], '607bc080dbb9', 'fresh']], ['o5', ['array', '<f4', [5], '51fb7d8c9563', 'fresh']], ['o6', ['array', '<i8', [7], '6984488c7681', 'fresh']], ['o7', ['array', '<f4', [5], '0310ddc723fc', 'fresh']], ['o8', ['array', '<i8', [7], '47f0a2d7b99f', 'fresh']], ['o9', ['array', '<f4', [5], '417230de77a6', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 1]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_parse_responses_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 10, 'result': ['ok', [[[['o0', ['array', '<i8', [7], '6984488c7681', 'fresh']], ['o1', ['array', '<f4', [5], '417230de77a6', 'fresh']], ['o2', ['array', '<i8', [7], '47f0a2d7b99f', 'fresh']], ['o3', ['array', '<f4', [5], 'c00c6de9a76d', 'fresh']], ['o4', ['array', '<i8', [7], '607bc080dbb9', 'fresh']], ['o5', ['array', '<f4', [5], '51fb7d8c9563', 'fresh']], ['o6', ['array', '<i8', [7], '6984488c7681', 'fresh']], ['o7', ['array', '<f4', [5], '0310ddc723fc', 'fresh']], ['o8', ['array', '<i8', [7], '47f0a2d7b99f', 'fresh']], ['o9', ['array', '<f4', [5], '417230de77a6', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 1]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_parse_responses_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 10, 'result': ['ok', [[[['o0', ['array', '<i8', [7], '6984488c7681', 'fresh']], ['o1', ['array', '<f4', [5], '417230de77a6', 'fresh']], ['o2', ['array', '<i8', [7], '47f0a2d7b99f', 'fresh']], ['o3', ['array', '<f4', [5], 'c00c6de9a76d', 'fresh']], ['o4', ['array', '<i8', [7], '607bc080dbb9', 'fresh']], ['o5', ['array', '<f4', [5], '51fb7d8c9563', 'fresh']], ['o6', ['array', '<i8', [7], '6984488c7681', 'fresh']], ['o7', ['array', '<f4', [5], '0310ddc723fc', 'fresh']], ['o8', ['array', '<i8', [7], '47f0a2d7b99f', 'fresh']], ['o9', ['array', '<f4', [5], '417230de77a6', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 1]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_parse_responses_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 10, 'result': ['ok', [[[['o0', ['array', '<i8', [7], '6984488c7681', 'fresh']], ['o1', ['array', '<f4', [5], '417230de77a6', 'fresh']], ['o2', ['array', '<i8', [7], '47f0a2d7b99f', 'fresh']], ['o3', ['array', '<f4', [5], 'c00c6de9a76d', 'fresh']], ['o4', ['array', '<i8', [7], '607bc080dbb9', 'fresh']], ['o5', ['array', '<f4', [5], '51fb7d8c9563', 'fresh']], ['o6', ['array', '<i8', [7], '6984488c7681', 'fresh']], ['o7', ['array', '<f4', [5], '0310ddc723fc', 'fresh']], ['o8', ['array', '<i8', [7], '47f0a2d7b99f', 'fresh']], ['o9', ['array', '<f4', [5], '417230de77a6', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 1]},
        ],
    },
    'decode_many_strict': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_parse_responses_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 3, 'result': ['ok', [[[['o0', ['array', '<f4', [5], '10f358f16a8b', 'fresh']], ['o1', ['array', '<f4', [5], 'df5a3f2b035e', 'fresh']], ['o2', ['array', '<f4', [5], '8f264031c27f', 'fresh']], ['o3', ['array', '<f4', [5], 'd52326878a3d', 'fresh']], ['o4', ['array', '<f4', [5], '9d03c78062f2', 'fresh']], ['o5', ['array', '<f4', [5], '5d3443a4d60e', 'fresh']], ['o6', ['array', '<f4', [5], '7caf92caf1a5', 'fresh']], ['o7', ['array', '<f4', [5], 'b1108aae2c65', 'fresh']], ['o8', ['array', '<f4', [5], '8215e6f03231', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 1]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_parse_responses_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 3, 'result': ['ok', [[[['o0', ['array', '<f4', [5], '10f358f16a8b', 'fresh']], ['o1', ['array', '<f4', [5], 'df5a3f2b035e', 'fresh']], ['o2', ['array', '<f4', [5], '8f264031c27f', 'fresh']], ['o3', ['array', '<f4', [5], 'd52326878a3d', 'fresh']], ['o4', ['array', '<f4', [5], '9d03c78062f2', 'fresh']], ['o5', ['array', '<f4', [5], '5d3443a4d60e', 'fresh']], ['o6', ['array', '<f4', [5], '7caf92caf1a5', 'fresh']], ['o7', ['array', '<f4', [5], 'b1108aae2c65', 'fresh']], ['o8', ['array', '<f4', [5], '8215e6f03231', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 1]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_parse_responses_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 3, 'result': ['ok', [[[['o0', ['array', '<f4', [5], '10f358f16a8b', 'fresh']], ['o1', ['array', '<f4', [5], 'df5a3f2b035e', 'fresh']], ['o2', ['array', '<f4', [5], '8f264031c27f', 'fresh']], ['o3', ['array', '<f4', [5], 'd52326878a3d', 'fresh']], ['o4', ['array', '<f4', [5], '9d03c78062f2', 'fresh']], ['o5', ['array', '<f4', [5], '5d3443a4d60e', 'fresh']], ['o6', ['array', '<f4', [5], '7caf92caf1a5', 'fresh']], ['o7', ['array', '<f4', [5], 'b1108aae2c65', 'fresh']], ['o8', ['array', '<f4', [5], '8215e6f03231', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 1]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_parse_responses_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 3, 'result': ['ok', [[[['o0', ['array', '<f4', [5], '10f358f16a8b', 'fresh']], ['o1', ['array', '<f4', [5], 'df5a3f2b035e', 'fresh']], ['o2', ['array', '<f4', [5], '8f264031c27f', 'fresh']], ['o3', ['array', '<f4', [5], 'd52326878a3d', 'fresh']], ['o4', ['array', '<f4', [5], '9d03c78062f2', 'fresh']], ['o5', ['array', '<f4', [5], '5d3443a4d60e', 'fresh']], ['o6', ['array', '<f4', [5], '7caf92caf1a5', 'fresh']], ['o7', ['array', '<f4', [5], 'b1108aae2c65', 'fresh']], ['o8', ['array', '<f4', [5], '8215e6f03231', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 1]},
        ],
    },
    'decode_many_tolerant': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_parse_responses_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 3, 'result': ['ok', [[[['o0', ['array', '<f4', [5], '10f358f16a8b', 'fresh']], ['o1', ['array', '<f4', [5], 'df5a3f2b035e', 'fresh']], ['o2', ['array', '<f4', [5], '8f264031c27f', 'fresh']], ['o3', ['array', '<f4', [5], 'd52326878a3d', 'fresh']], ['o4', ['array', '<f4', [5], '9d03c78062f2', 'fresh']], ['o5', ['array', '<f4', [5], '5d3443a4d60e', 'fresh']], ['o6', ['array', '<f4', [5], '7caf92caf1a5', 'fresh']], ['o7', ['array', '<f4', [5], 'b1108aae2c65', 'fresh']], ['o8', ['array', '<f4', [5], '8215e6f03231', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 1]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_parse_responses_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 3, 'result': ['ok', [[[['o0', ['array', '<f4', [5], '10f358f16a8b', 'fresh']], ['o1', ['array', '<f4', [5], 'df5a3f2b035e', 'fresh']], ['o2', ['array', '<f4', [5], '8f264031c27f', 'fresh']], ['o3', ['array', '<f4', [5], 'd52326878a3d', 'fresh']], ['o4', ['array', '<f4', [5], '9d03c78062f2', 'fresh']], ['o5', ['array', '<f4', [5], '5d3443a4d60e', 'fresh']], ['o6', ['array', '<f4', [5], '7caf92caf1a5', 'fresh']], ['o7', ['array', '<f4', [5], 'b1108aae2c65', 'fresh']], ['o8', ['array', '<f4', [5], '8215e6f03231', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 1]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_parse_responses_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 3, 'result': ['ok', [[[['o0', ['array', '<f4', [5], '10f358f16a8b', 'fresh']], ['o1', ['array', '<f4', [5], 'df5a3f2b035e', 'fresh']], ['o2', ['array', '<f4', [5], '8f264031c27f', 'fresh']], ['o3', ['array', '<f4', [5], 'd52326878a3d', 'fresh']], ['o4', ['array', '<f4', [5], '9d03c78062f2', 'fresh']], ['o5', ['array', '<f4', [5], '5d3443a4d60e', 'fresh']], ['o6', ['array', '<f4', [5], '7caf92caf1a5', 'fresh']], ['o7', ['array', '<f4', [5], 'b1108aae2c65', 'fresh']], ['o8', ['array', '<f4', [5], '8215e6f03231', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 1]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_parse_responses_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 3, 'result': ['ok', [[[['o0', ['array', '<f4', [5], '10f358f16a8b', 'fresh']], ['o1', ['array', '<f4', [5], 'df5a3f2b035e', 'fresh']], ['o2', ['array', '<f4', [5], '8f264031c27f', 'fresh']], ['o3', ['array', '<f4', [5], 'd52326878a3d', 'fresh']], ['o4', ['array', '<f4', [5], '9d03c78062f2', 'fresh']], ['o5', ['array', '<f4', [5], '5d3443a4d60e', 'fresh']], ['o6', ['array', '<f4', [5], '7caf92caf1a5', 'fresh']], ['o7', ['array', '<f4', [5], 'b1108aae2c65', 'fresh']], ['o8', ['array', '<f4', [5], '8215e6f03231', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 1]},
        ],
    },
    'decode_mixed_strict': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 3, 'result': ['ok', [[[['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['d', ['array', '<f8', [3, 1], '7f0639ce5dac', 'view']], ['classes', ['array', '<i8', [8, 5], '431851990268', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['classes', ['array', '<i8', [8, 5], '431851990268', 'view']], ['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['d', ['array', '<f8', [3, 1], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['classes', ['array', '<i8', [8, 5], '431851990268', 'view']], ['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['d', ['array', '<f8', [3, 1], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['classes', ['array', '<i8', [8, 5], '431851990268', 'view']], ['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['d', ['array', '<f8', [3, 1], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_mixed_tolerant': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['d', ['array', '<f8', [3, 1], '7f0639ce5dac', 'view']], ['classes', ['array', '<i8', [8, 5], '431851990268', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['classes', ['array', '<i8', [8, 5], '431851990268', 'view']], ['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['d', ['array', '<f8', [3, 1], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['classes', ['array', '<i8', [8, 5], '431851990268', 'view']], ['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['d', ['array', '<f8', [3, 1], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['classes', ['array', '<i8', [8, 5], '431851990268', 'view']], ['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['d', ['array', '<f8', [3, 1], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_one_strict': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['y', ['array', '<f4', [64, 33], '85fc1075c812', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['y', ['array', '<f4', [64, 33], '85fc1075c812', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['y', ['array', '<f4', [64, 33], '85fc1075c812', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['y', ['array', '<f4', [64, 33], '85fc1075c812', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_one_tolerant': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['y', ['array', '<f4', [64, 33], '85fc1075c812', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['y', ['array', '<f4', [64, 33], '85fc1075c812', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['y', ['array', '<f4', [64, 33], '85fc1075c812', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['y', ['array', '<f4', [64, 33], '85fc1075c812', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_pad_strict': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_pad_tolerant': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 3, 'result': ['ok', [[[['p', ['array', '<f4', [6], '307d2684464b', 'fresh']], ['z', ['array', '<f4', [4], 'e129f27c5103', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 3, 'result': ['ok', [[[['p', ['array', '<f4', [6], '307d2684464b', 'fresh']], ['z', ['array', '<f4', [4], 'e129f27c5103', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 3, 'result': ['ok', [[[['p', ['array', '<f4', [6], '307d2684464b', 'fresh']], ['z', ['array', '<f4', [4], 'e129f27c5103', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 3, 'result': ['ok', [[[['p', ['array', '<f4', [6], '307d2684464b', 'fresh']], ['z', ['array', '<f4', [4], 'e129f27c5103', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_rank0_strict': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'TypeError'], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'TypeError'], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'TypeError'], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'TypeError'], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_rank0_tolerant': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['r', ['array', '<f4', [], '7a28d220b360', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['r', ['array', '<f4', [], '7a28d220b360', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['r', ['array', '<f4', [], '7a28d220b360', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['r', ['array', '<f4', [], '7a28d220b360', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_strings_strict': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 3, 'result': ['ok', [[[['a', ['array', '<f4', [4], '8f6809c988e5', 'view']], ['s', ['array', '<U3', [2], '1424e0e98d55', 'fresh']], ['ids', ['array', '<i8', [6], '2b33b5254d22', 'fresh']], ['m', ['array', '|b1', [5], '78385b49bf10', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['a', ['array', '<f4', [4], '8f6809c988e5', 'view']], ['ids', ['array', '<i8', [6], '2b33b5254d22', 'view']], ['m', ['array', '|b1', [5], '78385b49bf10', 'view']], ['s', ['array', '<U3', [2], '1424e0e98d55', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['a', ['array', '<f4', [4], '8f6809c988e5', 'view']], ['ids', ['array', '<i8', [6], '2b33b5254d22', 'view']], ['m', ['array', '|b1', [5], '78385b49bf10', 'view']], ['s', ['array', '<U3', [2], '1424e0e98d55', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['a', ['array', '<f4', [4], '8f6809c988e5', 'view']], ['ids', ['array', '<i8', [6], '2b33b5254d22', 'view']], ['m', ['array', '|b1', [5], '78385b49bf10', 'view']], ['s', ['array', '<U3', [2], '1424e0e98d55', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_strings_tolerant': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 5, 'result': ['ok', [[[['a', ['array', '<f4', [4], '8f6809c988e5', 'view']], ['s', ['array', '<U3', [2], '1424e0e98d55', 'fresh']], ['ids', ['array', '<i8', [6], '2b33b5254d22', 'fresh']], ['m', ['array', '|b1', [5], '78385b49bf10', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['a', ['array', '<f4', [4], '8f6809c988e5', 'view']], ['ids', ['array', '<i8', [6], '2b33b5254d22', 'view']], ['m', ['array', '|b1', [5], '78385b49bf10', 'view']], ['s', ['array', '<U3', [2], '1424e0e98d55', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['a', ['array', '<f4', [4], '8f6809c988e5', 'view']], ['ids', ['array', '<i8', [6], '2b33b5254d22', 'view']], ['m', ['array', '|b1', [5], '78385b49bf10', 'view']], ['s', ['array', '<U3', [2], '1424e0e98d55', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['a', ['array', '<f4', [4], '8f6809c988e5', 'view']], ['ids', ['array', '<i8', [6], '2b33b5254d22', 'view']], ['m', ['array', '|b1', [5], '78385b49bf10', 'view']], ['s', ['array', '<U3', [2], '1424e0e98d55', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_tf_content_strict': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_tf_content_tolerant': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 2, 'result': ['ok', [[[['f', ['array', '<f4', [2], 'd151dee9298d', 'view']], ['c', ['array', '<f4', [2, 4], 'bdb1102548a0', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 2, 'result': ['ok', [[[['f', ['array', '<f4', [2], 'd151dee9298d', 'view']], ['c', ['array', '<f4', [2, 4], 'bdb1102548a0', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 2, 'result': ['ok', [[[['f', ['array', '<f4', [2], 'd151dee9298d', 'view']], ['c', ['array', '<f4', [2, 4], 'bdb1102548a0', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 2, 'result': ['ok', [[[['f', ['array', '<f4', [2], 'd151dee9298d', 'view']], ['c', ['array', '<f4', [2, 4], 'bdb1102548a0', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_truncated_strict': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_parse_responses_host': 1}, 'concat_device_calls': 0, 'launches': 2, 'result': ['raise', 'DecodeError'], 'seen_varints': False, 'stats': [0, 0, 1]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_parse_responses_host': 1}, 'concat_device_calls': 0, 'launches': 2, 'result': ['raise', 'DecodeError'], 'seen_varints': False, 'stats': [0, 0, 1]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_parse_responses_host': 1}, 'concat_device_calls': 0, 'launches': 2, 'result': ['raise', 'DecodeError'], 'seen_varints': True, 'stats': [0, 0, 1]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_parse_responses_host': 1}, 'concat_device_calls': 0, 'launches': 2, 'result': ['raise', 'DecodeError'], 'seen_varints': True, 'stats': [0, 0, 1]},
        ],
    },
    'decode_truncated_tolerant': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_parse_responses_host': 1}, 'concat_device_calls': 0, 'launches': 2, 'result': ['raise', 'DecodeError'], 'seen_varints': False, 'stats': [0, 0, 1]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_parse_responses_host': 1}, 'concat_device_calls': 0, 'launches': 2, 'result': ['raise', 'DecodeError'], 'seen_varints': False, 'stats': [0, 0, 1]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_parse_responses_host': 1}, 'concat_device_calls': 0, 'launches': 2, 'result': ['raise', 'DecodeError'], 'seen_varints': True, 'stats': [0, 0, 1]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_parse_responses_host': 1}, 'concat_device_calls': 0, 'launches': 2, 'result': ['raise', 'DecodeError'], 'seen_varints': True, 'stats': [0, 0, 1]},
        ],
    },
    'decode_varint_few_strict': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_varint_few_tolerant': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['x', ['array', '<i8', [4], 'e76ec5b00f39', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['x', ['array', '<i8', [4], 'e76ec5b00f39', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['x', ['array', '<i8', [4], 'e76ec5b00f39', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['x', ['array', '<i8', [4], 'e76ec5b00f39', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_varint_half_strict': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 3, 'result': ['ok', [[[['x', ['array', '<f2', [2], '78279d4f8280', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[[['x', ['array', '<f2', [2], '78279d4f8280', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[[['x', ['array', '<f2', [2], '78279d4f8280', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[[['x', ['array', '<f2', [2], '78279d4f8280', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_varint_half_tolerant': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['x', ['array', '<f2', [2], 'e8531aa90620', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['x', ['array', '<f2', [2], 'e8531aa90620', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['x', ['array', '<f2', [2], 'e8531aa90620', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['x', ['array', '<f2', [2], 'e8531aa90620', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_varint_parse_strict': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 3, 'result': ['raise', 'DecodeError'], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['raise', 'DecodeError'], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['raise', 'DecodeError'], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['raise', 'DecodeError'], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_varint_parse_tolerant': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 4, 'result': ['raise', 'DecodeError'], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 7, 'result': ['raise', 'DecodeError'], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 7, 'result': ['raise', 'DecodeError'], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 7, 'result': ['raise', 'DecodeError'], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_varint_range_strict': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 3, 'result': ['raise', 'OverflowError'], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['raise', 'OverflowError'], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['raise', 'OverflowError'], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['raise', 'OverflowError'], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_varint_range_tolerant': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 4, 'result': ['raise', 'OverflowError'], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 7, 'result': ['raise', 'OverflowError'], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 7, 'result': ['raise', 'OverflowError'], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 7, 'result': ['raise', 'OverflowError'], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_varint_rows_strict': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['x', ['array', '<i4', [3], '32e085535bb0', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 1]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 7, 'result': ['ok', [[[['x', ['array', '<i4', [3], '32e085535bb0', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 1]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 7, 'result': ['ok', [[[['x', ['array', '<i4', [3], '32e085535bb0', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 1]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 7, 'result': ['ok', [[[['x', ['array', '<i4', [3], '32e085535bb0', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 1]},
        ],
    },
    'decode_varint_rows_tolerant': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 5, 'result': ['ok', [[[['x', ['array', '<i4', [3], '32e085535bb0', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 1]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 8, 'result': ['ok', [[[['x', ['array', '<i4', [3], '32e085535bb0', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 1]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 8, 'result': ['ok', [[[['x', ['array', '<i4', [3], '32e085535bb0', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 1]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 8, 'result': ['ok', [[[['x', ['array', '<i4', [3], '32e085535bb0', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 1]},
        ],
    },
    'decode_varint_strict': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 3, 'result': ['ok', [[[['ids', ['array', '<i8', [3, 7], '52cb4304056a', 'fresh']], ['mask', ['array', '|b1', [9], '4f8cb9968539', 'fresh']], ['small', ['array', '<i4', [5], '430c389090db', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['ids', ['array', '<i8', [3, 7], '52cb4304056a', 'view']], ['mask', ['array', '|b1', [9], '4f8cb9968539', 'view']], ['small', ['array', '<i4', [5], '430c389090db', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['ids', ['array', '<i8', [3, 7], '52cb4304056a', 'view']], ['mask', ['array', '|b1', [9], '4f8cb9968539', 'view']], ['small', ['array', '<i4', [5], '430c389090db', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['ids', ['array', '<i8', [3, 7], '52cb4304056a', 'view']], ['mask', ['array', '|b1', [9], '4f8cb9968539', 'view']], ['small', ['array', '<i4', [5], '430c389090db', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_varint_tolerant': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[[['ids', ['array', '<i8', [3, 7], '52cb4304056a', 'fresh']], ['mask', ['array', '|b1', [9], '4f8cb9968539', 'fresh']], ['small', ['array', '<i4', [5], '430c389090db', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['ids', ['array', '<i8', [3, 7], '52cb4304056a', 'view']], ['mask', ['array', '|b1', [9], '4f8cb9968539', 'view']], ['small', ['array', '<i4', [5], '430c389090db', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['ids', ['array', '<i8', [3, 7], '52cb4304056a', 'view']], ['mask', ['array', '|b1', [9], '4f8cb9968539', 'view']], ['small', ['array', '<i4', [5], '430c389090db', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['ids', ['array', '<i8', [3, 7], '52cb4304056a', 'view']], ['mask', ['array', '|b1', [9], '4f8cb9968539', 'view']], ['small', ['array', '<i4', [5], '430c389090db', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_zero_none_strict': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['y', ['array', '<f4', [0], 'da39a3ee5e6b', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['y', ['array', '<f4', [0], 'da39a3ee5e6b', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['y', ['array', '<f4', [0], 'da39a3ee5e6b', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['y', ['array', '<f4', [0], 'da39a3ee5e6b', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_zero_none_tolerant': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['y', ['array', '<f4', [0], 'da39a3ee5e6b', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['y', ['array', '<f4', [0], 'da39a3ee5e6b', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['y', ['array', '<f4', [0], 'da39a3ee5e6b', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['y', ['array', '<f4', [0], 'da39a3ee5e6b', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_zero_run_strict': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['y', ['array', '<f4', [0], 'da39a3ee5e6b', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['y', ['array', '<f4', [0], 'da39a3ee5e6b', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['y', ['array', '<f4', [0], 'da39a3ee5e6b', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['y', ['array', '<f4', [0], 'da39a3ee5e6b', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_zero_run_tolerant': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['y', ['array', '<f4', [0], 'da39a3ee5e6b', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['y', ['array', '<f4', [0], 'da39a3ee5e6b', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['y', ['array', '<f4', [0], 'da39a3ee5e6b', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['y', ['array', '<f4', [0], 'da39a3ee5e6b', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_zero_varint_strict': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['v', ['array', '<i8', [0], 'da39a3ee5e6b', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['v', ['array', '<i8', [0], 'da39a3ee5e6b', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['v', ['array', '<i8', [0], 'da39a3ee5e6b', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['v', ['array', '<i8', [0], 'da39a3ee5e6b', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'decode_zero_varint_tolerant': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['v', ['array', '<i8', [0], 'da39a3ee5e6b', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['v', ['array', '<i8', [0], 'da39a3ee5e6b', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['v', ['array', '<i8', [0], 'da39a3ee5e6b', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['v', ['array', '<i8', [0], 'da39a3ee5e6b', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'narrow_bf16_full': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_set_decode_cast': 2}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['f', ['array', '<V2', [30, 7], 'f089677fa26e', 'view']], ['g', ['array', '<V2', [99], 'ef86e6719f9b', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['f', ['array', '<V2', [30, 7], 'f089677fa26e', 'view']], ['g', ['array', '<V2', [99], 'ef86e6719f9b', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [2, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_set_decode_cast': 2}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['f', ['array', '<V2', [30, 7], 'f089677fa26e', 'view']], ['g', ['array', '<V2', [99], 'ef86e6719f9b', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['f', ['array', '<V2', [30, 7], 'f089677fa26e', 'view']], ['g', ['array', '<V2', [99], 'ef86e6719f9b', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [2, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_cast': 2}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['f', ['array', '<V2', [30, 7], 'f089677fa26e', 'view']], ['g', ['array', '<V2', [99], 'ef86e6719f9b', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['f', ['array', '<V2', [30, 7], 'f089677fa26e', 'view']], ['g', ['array', '<V2', [99], 'ef86e6719f9b', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [2, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_cast': 2}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[[['f', ['array', '<V2', [30, 7], 'f089677fa26e', 'view']], ['g', ['array', '<V2', [99], 'ef86e6719f9b', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']], [[['f', ['array', '<V2', [30, 7], 'f089677fa26e', 'view']], ['g', ['array', '<V2', [99], 'ef86e6719f9b', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [2, 0, 0]},
        ],
    },
    'narrow_f16_and_ids': {
        'cold': [
            {'calls': {'b200tfs_parse_responses_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_parse_responses_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_parse_responses_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_parse_responses_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'narrow_f16_full': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_set_decode_cast': 2, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['f', ['array', '<f2', [30, 7], '3fcbd8357a1d', 'view']], ['g', ['array', '<f2', [99], '5cad6c916a70', 'view']], ['ids', ['array', '<i8', [50], '4b1051119c86', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_cast': 2, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['f', ['array', '<f2', [30, 7], '3fcbd8357a1d', 'view']], ['g', ['array', '<f2', [99], '5cad6c916a70', 'view']], ['ids', ['array', '<i8', [50], '4b1051119c86', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_cast': 2, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['f', ['array', '<f2', [30, 7], '3fcbd8357a1d', 'view']], ['g', ['array', '<f2', [99], '5cad6c916a70', 'view']], ['ids', ['array', '<i8', [50], '4b1051119c86', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_cast': 2, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['f', ['array', '<f2', [30, 7], '3fcbd8357a1d', 'view']], ['g', ['array', '<f2', [99], '5cad6c916a70', 'view']], ['ids', ['array', '<i8', [50], '4b1051119c86', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'narrow_f16_full_strict': {
        'cold': [
            {'calls': {'b200tfs_parse_responses_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['f', ['array', '<f2', [30, 7], '3fcbd8357a1d', 'fresh']], ['g', ['array', '<f2', [99], '5cad6c916a70', 'fresh']], ['ids', ['array', '<i8', [50], '4b1051119c86', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_parse_responses_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['f', ['array', '<f2', [30, 7], '3fcbd8357a1d', 'fresh']], ['g', ['array', '<f2', [99], '5cad6c916a70', 'fresh']], ['ids', ['array', '<i8', [50], '4b1051119c86', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_parse_responses_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['f', ['array', '<f2', [30, 7], '3fcbd8357a1d', 'fresh']], ['g', ['array', '<f2', [99], '5cad6c916a70', 'fresh']], ['ids', ['array', '<i8', [50], '4b1051119c86', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_parse_responses_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[[['f', ['array', '<f2', [30, 7], '3fcbd8357a1d', 'fresh']], ['g', ['array', '<f2', [99], '5cad6c916a70', 'fresh']], ['ids', ['array', '<i8', [50], '4b1051119c86', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'narrow_f16_padding': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_set_decode_cast': 2}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_set_decode_cast': 2}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_cast': 2}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_cast': 2}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'narrow_f16_partial': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_parse_responses_host': 1, 'b200tfs_set_decode_cast': 2, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[[['f', ['array', '<f2', [30, 7], '3fcbd8357a1d', 'fresh']], ['g', ['array', '<f4', [99], '13896d92b1df', 'fresh']], ['ids', ['array', '<i8', [50], '4b1051119c86', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_parse_responses_host': 1, 'b200tfs_set_decode_cast': 2, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[[['f', ['array', '<f2', [30, 7], '3fcbd8357a1d', 'fresh']], ['g', ['array', '<f4', [99], '13896d92b1df', 'fresh']], ['ids', ['array', '<i8', [50], '4b1051119c86', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_parse_responses_host': 1, 'b200tfs_set_decode_cast': 2, 'b200tfs_set_decode_varints': 2, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 9, 'result': ['ok', [[[['f', ['array', '<f2', [30, 7], '3fcbd8357a1d', 'fresh']], ['g', ['array', '<f4', [99], '13896d92b1df', 'fresh']], ['ids', ['array', '<i8', [50], '4b1051119c86', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_parse_responses_host': 1, 'b200tfs_set_decode_cast': 2, 'b200tfs_set_decode_varints': 2, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 9, 'result': ['ok', [[[['f', ['array', '<f2', [30, 7], '3fcbd8357a1d', 'fresh']], ['g', ['array', '<f4', [99], '13896d92b1df', 'fresh']], ['ids', ['array', '<i8', [50], '4b1051119c86', 'fresh']]], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'open_bf16': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['b', [['ok', None], ['ok', None], ['ok', None], '0bed4a5a280d']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [['b', [['ok', ['array', '<V2', [2], '18d36867d977', 'view']], ['raise', 'KeyError'], ['ok', ['array', '<V2', [2], '18d36867d977', 'fresh']], '0bed4a5a280d']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [['b', [['ok', ['array', '<V2', [2], '18d36867d977', 'view']], ['raise', 'KeyError'], ['ok', ['array', '<V2', [2], '18d36867d977', 'fresh']], '0bed4a5a280d']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [['b', [['ok', ['array', '<V2', [2], '18d36867d977', 'view']], ['raise', 'KeyError'], ['ok', ['array', '<V2', [2], '18d36867d977', 'fresh']], '0bed4a5a280d']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'open_complex': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['c', [['ok', ['array', '<c8', [2], '30c3c8e10060', 'view']], ['raise', 'ValueError'], ['ok', ['array', '<c8', [2], '30c3c8e10060', 'fresh']], '5cd87a1f161b']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['c', [['ok', ['array', '<c8', [2], '30c3c8e10060', 'view']], ['raise', 'ValueError'], ['ok', ['array', '<c8', [2], '30c3c8e10060', 'fresh']], '5cd87a1f161b']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['c', [['ok', ['array', '<c8', [2], '30c3c8e10060', 'view']], ['raise', 'ValueError'], ['ok', ['array', '<c8', [2], '30c3c8e10060', 'fresh']], '5cd87a1f161b']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['c', [['ok', ['array', '<c8', [2], '30c3c8e10060', 'view']], ['raise', 'ValueError'], ['ok', ['array', '<c8', [2], '30c3c8e10060', 'fresh']], '5cd87a1f161b']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'open_content': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['c', [['ok', None], ['ok', None], ['ok', None], '00bbd7234c65']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['c', [['ok', None], ['ok', None], ['ok', None], '00bbd7234c65']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['c', [['ok', None], ['ok', None], ['ok', None], '00bbd7234c65']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['c', [['ok', None], ['ok', None], ['ok', None], '00bbd7234c65']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'open_empty': {
        'cold': [
            {'calls': {}, 'concat_device_calls': 0, 'launches': 0, 'result': ['ok', None], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {}, 'concat_device_calls': 0, 'launches': 0, 'result': ['ok', None], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {}, 'concat_device_calls': 0, 'launches': 0, 'result': ['ok', None], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {}, 'concat_device_calls': 0, 'launches': 0, 'result': ['ok', None], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'open_flipped': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['d', [['ok', ['array', '<f8', [3], '7f0639ce5dac', 'view']], ['ok', ['array', '<f8', [3], '7f0639ce5dac', 'fresh']], ['ok', ['array', '<f8', [3], '7f0639ce5dac', 'fresh']], '84b8033be190']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['d', [['ok', ['array', '<f8', [3], '7f0639ce5dac', 'view']], ['ok', ['array', '<f8', [3], '7f0639ce5dac', 'fresh']], ['ok', ['array', '<f8', [3], '7f0639ce5dac', 'fresh']], '84b8033be190']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['d', [['ok', ['array', '<f8', [3], '7f0639ce5dac', 'view']], ['ok', ['array', '<f8', [3], '7f0639ce5dac', 'fresh']], ['ok', ['array', '<f8', [3], '7f0639ce5dac', 'fresh']], '84b8033be190']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['d', [['ok', ['array', '<f8', [3], '7f0639ce5dac', 'view']], ['ok', ['array', '<f8', [3], '7f0639ce5dac', 'fresh']], ['ok', ['array', '<f8', [3], '7f0639ce5dac', 'fresh']], '84b8033be190']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'open_floats': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['scores', [['ok', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['ok', ['array', '<f4', [8, 5], '640ba4d3c6af', 'fresh']], ['ok', ['array', '<f4', [8, 5], '640ba4d3c6af', 'fresh']], '41a1c2041200']], ['d', [['ok', ['array', '<f8', [3], '7f0639ce5dac', 'view']], ['ok', ['array', '<f8', [3], '7f0639ce5dac', 'fresh']], ['ok', ['array', '<f8', [3], '7f0639ce5dac', 'fresh']], '84b8033be190']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['scores', [['ok', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['ok', ['array', '<f4', [8, 5], '640ba4d3c6af', 'fresh']], ['ok', ['array', '<f4', [8, 5], '640ba4d3c6af', 'fresh']], '41a1c2041200']], ['d', [['ok', ['array', '<f8', [3], '7f0639ce5dac', 'view']], ['ok', ['array', '<f8', [3], '7f0639ce5dac', 'fresh']], ['ok', ['array', '<f8', [3], '7f0639ce5dac', 'fresh']], '84b8033be190']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['scores', [['ok', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['ok', ['array', '<f4', [8, 5], '640ba4d3c6af', 'fresh']], ['ok', ['array', '<f4', [8, 5], '640ba4d3c6af', 'fresh']], '41a1c2041200']], ['d', [['ok', ['array', '<f8', [3], '7f0639ce5dac', 'view']], ['ok', ['array', '<f8', [3], '7f0639ce5dac', 'fresh']], ['ok', ['array', '<f8', [3], '7f0639ce5dac', 'fresh']], '84b8033be190']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['scores', [['ok', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['ok', ['array', '<f4', [8, 5], '640ba4d3c6af', 'fresh']], ['ok', ['array', '<f4', [8, 5], '640ba4d3c6af', 'fresh']], '41a1c2041200']], ['d', [['ok', ['array', '<f8', [3], '7f0639ce5dac', 'view']], ['ok', ['array', '<f8', [3], '7f0639ce5dac', 'fresh']], ['ok', ['array', '<f8', [3], '7f0639ce5dac', 'fresh']], '84b8033be190']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'open_half': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['h', [['ok', None], ['ok', None], ['ok', None], 'b8aa5c97b5ac']], ['f', [['ok', ['array', '<f4', [5], '10f358f16a8b', 'view']], ['ok', ['array', '<f4', [5], '10f358f16a8b', 'fresh']], ['ok', ['array', '<f4', [5], '10f358f16a8b', 'fresh']], '44adb024c18a']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [['h', [['ok', ['array', '<f2', [6], '8a8ce3354514', 'view']], ['ok', None], ['ok', ['array', '<f2', [6], '8a8ce3354514', 'fresh']], 'b8aa5c97b5ac']], ['f', [['ok', ['array', '<f4', [5], '10f358f16a8b', 'view']], ['ok', ['array', '<f4', [5], '10f358f16a8b', 'fresh']], ['ok', ['array', '<f4', [5], '10f358f16a8b', 'fresh']], '44adb024c18a']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [['h', [['ok', ['array', '<f2', [6], '8a8ce3354514', 'view']], ['ok', None], ['ok', ['array', '<f2', [6], '8a8ce3354514', 'fresh']], 'b8aa5c97b5ac']], ['f', [['ok', ['array', '<f4', [5], '10f358f16a8b', 'view']], ['ok', ['array', '<f4', [5], '10f358f16a8b', 'fresh']], ['ok', ['array', '<f4', [5], '10f358f16a8b', 'fresh']], '44adb024c18a']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [['h', [['ok', ['array', '<f2', [6], '8a8ce3354514', 'view']], ['ok', None], ['ok', ['array', '<f2', [6], '8a8ce3354514', 'fresh']], 'b8aa5c97b5ac']], ['f', [['ok', ['array', '<f4', [5], '10f358f16a8b', 'view']], ['ok', ['array', '<f4', [5], '10f358f16a8b', 'fresh']], ['ok', ['array', '<f4', [5], '10f358f16a8b', 'fresh']], '44adb024c18a']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'open_many': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', None], 'seen_varints': False, 'stats': [0, 0, 1]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', None], 'seen_varints': False, 'stats': [0, 0, 1]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', None], 'seen_varints': True, 'stats': [0, 0, 1]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', None], 'seen_varints': True, 'stats': [0, 0, 1]},
        ],
    },
    'open_many_mixed': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', None], 'seen_varints': False, 'stats': [0, 0, 1]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', None], 'seen_varints': False, 'stats': [0, 0, 1]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', None], 'seen_varints': True, 'stats': [0, 0, 1]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', None], 'seen_varints': True, 'stats': [0, 0, 1]},
        ],
    },
    'open_mixed': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['classes', [['ok', None], ['ok', None], ['ok', None], '27acd729deb7']], ['scores', [['ok', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['ok', ['array', '<f4', [8, 5], '640ba4d3c6af', 'fresh']], ['ok', ['array', '<f4', [8, 5], '640ba4d3c6af', 'fresh']], '41a1c2041200']], ['d', [['ok', ['array', '<f8', [3, 1], '7f0639ce5dac', 'view']], ['ok', ['array', '<f8', [3, 1], '7f0639ce5dac', 'fresh']], ['ok', ['array', '<f8', [3, 1], '7f0639ce5dac', 'fresh']], '4ca811446030']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [['classes', [['ok', ['array', '<i8', [8, 5], '431851990268', 'view']], ['ok', ['array', '<i8', [8, 5], '431851990268', 'fresh']], ['ok', ['array', '<i8', [8, 5], '431851990268', 'fresh']], '27acd729deb7']], ['scores', [['ok', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['ok', ['array', '<f4', [8, 5], '640ba4d3c6af', 'fresh']], ['ok', ['array', '<f4', [8, 5], '640ba4d3c6af', 'fresh']], '41a1c2041200']], ['d', [['ok', ['array', '<f8', [3, 1], '7f0639ce5dac', 'view']], ['ok', ['array', '<f8', [3, 1], '7f0639ce5dac', 'fresh']], ['ok', ['array', '<f8', [3, 1], '7f0639ce5dac', 'fresh']], '4ca811446030']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [['classes', [['ok', ['array', '<i8', [8, 5], '431851990268', 'view']], ['ok', ['array', '<i8', [8, 5], '431851990268', 'fresh']], ['ok', ['array', '<i8', [8, 5], '431851990268', 'fresh']], '27acd729deb7']], ['scores', [['ok', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['ok', ['array', '<f4', [8, 5], '640ba4d3c6af', 'fresh']], ['ok', ['array', '<f4', [8, 5], '640ba4d3c6af', 'fresh']], '41a1c2041200']], ['d', [['ok', ['array', '<f8', [3, 1], '7f0639ce5dac', 'view']], ['ok', ['array', '<f8', [3, 1], '7f0639ce5dac', 'fresh']], ['ok', ['array', '<f8', [3, 1], '7f0639ce5dac', 'fresh']], '4ca811446030']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [['classes', [['ok', ['array', '<i8', [8, 5], '431851990268', 'view']], ['ok', ['array', '<i8', [8, 5], '431851990268', 'fresh']], ['ok', ['array', '<i8', [8, 5], '431851990268', 'fresh']], '27acd729deb7']], ['scores', [['ok', ['array', '<f4', [8, 5], '640ba4d3c6af', 'view']], ['ok', ['array', '<f4', [8, 5], '640ba4d3c6af', 'fresh']], ['ok', ['array', '<f4', [8, 5], '640ba4d3c6af', 'fresh']], '41a1c2041200']], ['d', [['ok', ['array', '<f8', [3, 1], '7f0639ce5dac', 'view']], ['ok', ['array', '<f8', [3, 1], '7f0639ce5dac', 'fresh']], ['ok', ['array', '<f8', [3, 1], '7f0639ce5dac', 'fresh']], '4ca811446030']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'open_one': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['y', [['ok', ['array', '<f4', [64, 33], '85fc1075c812', 'view']], ['ok', ['array', '<f4', [64, 33], '85fc1075c812', 'fresh']], ['ok', ['array', '<f4', [64, 33], '85fc1075c812', 'fresh']], 'a95e6d378096']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['y', [['ok', ['array', '<f4', [64, 33], '85fc1075c812', 'view']], ['ok', ['array', '<f4', [64, 33], '85fc1075c812', 'fresh']], ['ok', ['array', '<f4', [64, 33], '85fc1075c812', 'fresh']], 'a95e6d378096']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['y', [['ok', ['array', '<f4', [64, 33], '85fc1075c812', 'view']], ['ok', ['array', '<f4', [64, 33], '85fc1075c812', 'fresh']], ['ok', ['array', '<f4', [64, 33], '85fc1075c812', 'fresh']], 'a95e6d378096']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['y', [['ok', ['array', '<f4', [64, 33], '85fc1075c812', 'view']], ['ok', ['array', '<f4', [64, 33], '85fc1075c812', 'fresh']], ['ok', ['array', '<f4', [64, 33], '85fc1075c812', 'fresh']], 'a95e6d378096']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'open_pad': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['p', [['ok', None], ['ok', None], ['ok', None], '212e97a8d658']], ['z', [['ok', None], ['ok', None], ['ok', None], '70e11885c033']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['p', [['ok', None], ['ok', None], ['ok', None], '212e97a8d658']], ['z', [['ok', None], ['ok', None], ['ok', None], '70e11885c033']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['p', [['ok', None], ['ok', None], ['ok', None], '212e97a8d658']], ['z', [['ok', None], ['ok', None], ['ok', None], '70e11885c033']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['p', [['ok', None], ['ok', None], ['ok', None], '212e97a8d658']], ['z', [['ok', None], ['ok', None], ['ok', None], '70e11885c033']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'open_rank0': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['r', [['ok', ['array', '<f4', [], '7a28d220b360', 'view']], ['raise', 'TypeError'], ['ok', ['array', '<f4', [], '7a28d220b360', 'fresh']], '30ff27575f03']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['r', [['ok', ['array', '<f4', [], '7a28d220b360', 'view']], ['raise', 'TypeError'], ['ok', ['array', '<f4', [], '7a28d220b360', 'fresh']], '30ff27575f03']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['r', [['ok', ['array', '<f4', [], '7a28d220b360', 'view']], ['raise', 'TypeError'], ['ok', ['array', '<f4', [], '7a28d220b360', 'fresh']], '30ff27575f03']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['r', [['ok', ['array', '<f4', [], '7a28d220b360', 'view']], ['raise', 'TypeError'], ['ok', ['array', '<f4', [], '7a28d220b360', 'fresh']], '30ff27575f03']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'open_strings': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['a', [['ok', ['array', '<f4', [4], '8f6809c988e5', 'view']], ['ok', ['array', '<f4', [4], '8f6809c988e5', 'fresh']], ['ok', ['array', '<f4', [4], '8f6809c988e5', 'fresh']], 'f68f675fa161']], ['ids', [['ok', None], ['ok', None], ['ok', None], '246b937fa671']], ['m', [['ok', None], ['ok', None], ['ok', None], 'abba4c061fc9']], ['s', [['ok', None], ['ok', None], ['ok', None], '7eefdf582f24']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [['a', [['ok', ['array', '<f4', [4], '8f6809c988e5', 'view']], ['ok', ['array', '<f4', [4], '8f6809c988e5', 'fresh']], ['ok', ['array', '<f4', [4], '8f6809c988e5', 'fresh']], 'f68f675fa161']], ['ids', [['ok', ['array', '<i8', [6], '2b33b5254d22', 'view']], ['ok', ['array', '<i8', [6], '2b33b5254d22', 'fresh']], ['ok', ['array', '<i8', [6], '2b33b5254d22', 'fresh']], '246b937fa671']], ['m', [['ok', ['array', '|b1', [5], '78385b49bf10', 'view']], ['ok', ['array', '|b1', [5], '78385b49bf10', 'fresh']], ['ok', ['array', '|b1', [5], '78385b49bf10', 'fresh']], 'abba4c061fc9']], ['s', [['ok', None], ['ok', None], ['ok', None], '7eefdf582f24']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [['a', [['ok', ['array', '<f4', [4], '8f6809c988e5', 'view']], ['ok', ['array', '<f4', [4], '8f6809c988e5', 'fresh']], ['ok', ['array', '<f4', [4], '8f6809c988e5', 'fresh']], 'f68f675fa161']], ['ids', [['ok', ['array', '<i8', [6], '2b33b5254d22', 'view']], ['ok', ['array', '<i8', [6], '2b33b5254d22', 'fresh']], ['ok', ['array', '<i8', [6], '2b33b5254d22', 'fresh']], '246b937fa671']], ['m', [['ok', ['array', '|b1', [5], '78385b49bf10', 'view']], ['ok', ['array', '|b1', [5], '78385b49bf10', 'fresh']], ['ok', ['array', '|b1', [5], '78385b49bf10', 'fresh']], 'abba4c061fc9']], ['s', [['ok', None], ['ok', None], ['ok', None], '7eefdf582f24']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [['a', [['ok', ['array', '<f4', [4], '8f6809c988e5', 'view']], ['ok', ['array', '<f4', [4], '8f6809c988e5', 'fresh']], ['ok', ['array', '<f4', [4], '8f6809c988e5', 'fresh']], 'f68f675fa161']], ['ids', [['ok', ['array', '<i8', [6], '2b33b5254d22', 'view']], ['ok', ['array', '<i8', [6], '2b33b5254d22', 'fresh']], ['ok', ['array', '<i8', [6], '2b33b5254d22', 'fresh']], '246b937fa671']], ['m', [['ok', ['array', '|b1', [5], '78385b49bf10', 'view']], ['ok', ['array', '|b1', [5], '78385b49bf10', 'fresh']], ['ok', ['array', '|b1', [5], '78385b49bf10', 'fresh']], 'abba4c061fc9']], ['s', [['ok', None], ['ok', None], ['ok', None], '7eefdf582f24']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'open_tf_content': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['c', [['ok', None], ['ok', None], ['ok', None], '2a0d9a8f8817']], ['f', [['ok', ['array', '<f4', [2], 'd151dee9298d', 'view']], ['ok', ['array', '<f4', [2], 'd151dee9298d', 'fresh']], ['ok', ['array', '<f4', [2], 'd151dee9298d', 'fresh']], '81bb65dc2df4']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['c', [['ok', None], ['ok', None], ['ok', None], '2a0d9a8f8817']], ['f', [['ok', ['array', '<f4', [2], 'd151dee9298d', 'view']], ['ok', ['array', '<f4', [2], 'd151dee9298d', 'fresh']], ['ok', ['array', '<f4', [2], 'd151dee9298d', 'fresh']], '81bb65dc2df4']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['c', [['ok', None], ['ok', None], ['ok', None], '2a0d9a8f8817']], ['f', [['ok', ['array', '<f4', [2], 'd151dee9298d', 'view']], ['ok', ['array', '<f4', [2], 'd151dee9298d', 'fresh']], ['ok', ['array', '<f4', [2], 'd151dee9298d', 'fresh']], '81bb65dc2df4']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['c', [['ok', None], ['ok', None], ['ok', None], '2a0d9a8f8817']], ['f', [['ok', ['array', '<f4', [2], 'd151dee9298d', 'view']], ['ok', ['array', '<f4', [2], 'd151dee9298d', 'fresh']], ['ok', ['array', '<f4', [2], 'd151dee9298d', 'fresh']], '81bb65dc2df4']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'open_truncated': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', None], 'seen_varints': False, 'stats': [0, 0, 1]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', None], 'seen_varints': False, 'stats': [0, 0, 1]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', None], 'seen_varints': True, 'stats': [0, 0, 1]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', None], 'seen_varints': True, 'stats': [0, 0, 1]},
        ],
    },
    'open_varint': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['ids', [['ok', None], ['ok', None], ['ok', None], '2fb365f9ba32']], ['mask', [['ok', None], ['ok', None], ['ok', None], '09395ebaff25']], ['small', [['ok', None], ['ok', None], ['ok', None], '76a39ee67e1c']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [['ids', [['ok', ['array', '<i8', [3, 7], '52cb4304056a', 'view']], ['ok', ['array', '<i8', [3, 7], '52cb4304056a', 'fresh']], ['ok', ['array', '<i8', [3, 7], '52cb4304056a', 'fresh']], '2fb365f9ba32']], ['mask', [['ok', ['array', '|b1', [9], '4f8cb9968539', 'view']], ['ok', ['array', '|b1', [9], '4f8cb9968539', 'fresh']], ['ok', ['array', '|b1', [9], '4f8cb9968539', 'fresh']], '09395ebaff25']], ['small', [['ok', ['array', '<i4', [5], '430c389090db', 'view']], ['ok', ['array', '<i4', [5], '430c389090db', 'fresh']], ['ok', ['array', '<i4', [5], '430c389090db', 'fresh']], '76a39ee67e1c']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [['ids', [['ok', ['array', '<i8', [3, 7], '52cb4304056a', 'view']], ['ok', ['array', '<i8', [3, 7], '52cb4304056a', 'fresh']], ['ok', ['array', '<i8', [3, 7], '52cb4304056a', 'fresh']], '2fb365f9ba32']], ['mask', [['ok', ['array', '|b1', [9], '4f8cb9968539', 'view']], ['ok', ['array', '|b1', [9], '4f8cb9968539', 'fresh']], ['ok', ['array', '|b1', [9], '4f8cb9968539', 'fresh']], '09395ebaff25']], ['small', [['ok', ['array', '<i4', [5], '430c389090db', 'view']], ['ok', ['array', '<i4', [5], '430c389090db', 'fresh']], ['ok', ['array', '<i4', [5], '430c389090db', 'fresh']], '76a39ee67e1c']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [['ids', [['ok', ['array', '<i8', [3, 7], '52cb4304056a', 'view']], ['ok', ['array', '<i8', [3, 7], '52cb4304056a', 'fresh']], ['ok', ['array', '<i8', [3, 7], '52cb4304056a', 'fresh']], '2fb365f9ba32']], ['mask', [['ok', ['array', '|b1', [9], '4f8cb9968539', 'view']], ['ok', ['array', '|b1', [9], '4f8cb9968539', 'fresh']], ['ok', ['array', '|b1', [9], '4f8cb9968539', 'fresh']], '09395ebaff25']], ['small', [['ok', ['array', '<i4', [5], '430c389090db', 'view']], ['ok', ['array', '<i4', [5], '430c389090db', 'fresh']], ['ok', ['array', '<i4', [5], '430c389090db', 'fresh']], '76a39ee67e1c']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'open_varint_few': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['x', [['ok', None], ['ok', None], ['ok', None], '39e560f4fbc9']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['x', [['ok', None], ['ok', None], ['ok', None], '39e560f4fbc9']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['x', [['ok', None], ['ok', None], ['ok', None], '39e560f4fbc9']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['x', [['ok', None], ['ok', None], ['ok', None], '39e560f4fbc9']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'open_varint_half': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['x', [['ok', None], ['ok', None], ['ok', None], '21945fdbaa5e']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [['x', [['ok', ['array', '<f2', [2], 'e8531aa90620', 'view']], ['ok', None], ['ok', ['array', '<f2', [2], 'e8531aa90620', 'fresh']], '21945fdbaa5e']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [['x', [['ok', ['array', '<f2', [2], 'e8531aa90620', 'view']], ['ok', None], ['ok', ['array', '<f2', [2], 'e8531aa90620', 'fresh']], '21945fdbaa5e']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [['x', [['ok', ['array', '<f2', [2], 'e8531aa90620', 'view']], ['ok', None], ['ok', ['array', '<f2', [2], 'e8531aa90620', 'fresh']], '21945fdbaa5e']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'open_varint_parse': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['x', [['ok', None], ['ok', None], ['ok', None], '3aaa0c9fb226']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [['x', [['ok', None], ['ok', None], ['ok', None], '3aaa0c9fb226']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [['x', [['ok', None], ['ok', None], ['ok', None], '3aaa0c9fb226']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [['x', [['ok', None], ['ok', None], ['ok', None], '3aaa0c9fb226']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'open_varint_range': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['x', [['ok', None], ['ok', None], ['ok', None], '8e900f199d6e']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [['x', [['ok', None], ['ok', None], ['ok', None], '8e900f199d6e']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [['x', [['ok', None], ['ok', None], ['ok', None], '8e900f199d6e']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [['x', [['ok', None], ['ok', None], ['ok', None], '8e900f199d6e']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'open_varint_rows': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['x', [['ok', None], ['ok', None], ['ok', None], '591ab42c3a49']]]], 'seen_varints': True, 'stats': [0, 0, 1]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [['x', [['ok', None], ['ok', None], ['ok', None], '591ab42c3a49']]]], 'seen_varints': True, 'stats': [0, 0, 1]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [['x', [['ok', None], ['ok', None], ['ok', None], '591ab42c3a49']]]], 'seen_varints': True, 'stats': [0, 0, 1]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [['x', [['ok', None], ['ok', None], ['ok', None], '591ab42c3a49']]]], 'seen_varints': True, 'stats': [0, 0, 1]},
        ],
    },
    'open_zero_none': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['y', [['ok', None], ['ok', None], ['ok', None], '57b29a684f93']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['y', [['ok', None], ['ok', None], ['ok', None], '57b29a684f93']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['y', [['ok', None], ['ok', None], ['ok', None], '57b29a684f93']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['y', [['ok', None], ['ok', None], ['ok', None], '57b29a684f93']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'open_zero_run': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['y', [['ok', None], ['ok', None], ['ok', None], '699a7159825d']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['y', [['ok', None], ['ok', None], ['ok', None], '699a7159825d']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['y', [['ok', None], ['ok', None], ['ok', None], '699a7159825d']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['y', [['ok', None], ['ok', None], ['ok', None], '699a7159825d']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'open_zero_varint': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['v', [['ok', None], ['ok', None], ['ok', None], '9af69703f53c']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['v', [['ok', None], ['ok', None], ['ok', None], '9af69703f53c']]]], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['v', [['ok', None], ['ok', None], ['ok', None], '9af69703f53c']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['v', [['ok', None], ['ok', None], ['ok', None], '9af69703f53c']]]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'out_numpy': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'out']], ['d', ['array', '<f8', [3, 1], '7f0639ce5dac', 'view']], ['classes', ['array', '<i8', [8, 5], '431851990268', 'out']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[['classes', ['array', '<i8', [8, 5], '431851990268', 'out']], ['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'out']], ['d', ['array', '<f8', [3, 1], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[['classes', ['array', '<i8', [8, 5], '431851990268', 'out']], ['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'out']], ['d', ['array', '<f8', [3, 1], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[['classes', ['array', '<i8', [8, 5], '431851990268', 'out']], ['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'out']], ['d', ['array', '<f8', [3, 1], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'out_numpy_mismatch': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 4, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'out_numpy_missing_key': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 4, 'result': ['raise', 'KeyError'], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['raise', 'KeyError'], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['raise', 'KeyError'], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['raise', 'KeyError'], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'out_numpy_one': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[['y', ['array', '<f4', [64, 33], '85fc1075c812', 'out']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[['y', ['array', '<f4', [64, 33], '85fc1075c812', 'out']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[['y', ['array', '<f4', [64, 33], '85fc1075c812', 'out']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[['y', ['array', '<f4', [64, 33], '85fc1075c812', 'out']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'out_pinned': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[['y', ['array', '<f4', [64, 33], '85fc1075c812', 'out']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[['y', ['array', '<f4', [64, 33], '85fc1075c812', 'out']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[['y', ['array', '<f4', [64, 33], '85fc1075c812', 'out']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[['y', ['array', '<f4', [64, 33], '85fc1075c812', 'out']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'out_pinned_dtype_mismatch': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 2, 'b200tfs_decode_results': 2}, 'concat_device_calls': 0, 'launches': 2, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [2, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 2, 'b200tfs_decode_results': 2}, 'concat_device_calls': 0, 'launches': 2, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [2, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 2, 'b200tfs_decode_results': 2, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 2, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [2, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 2, 'b200tfs_decode_results': 2, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 2, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [2, 0, 0]},
        ],
    },
    'out_pinned_f64': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[['y', ['array', '<f8', [3], '7f0639ce5dac', 'out']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[['y', ['array', '<f8', [3], '7f0639ce5dac', 'out']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[['y', ['array', '<f8', [3], '7f0639ce5dac', 'out']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[['y', ['array', '<f8', [3], '7f0639ce5dac', 'out']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'out_pinned_missing_key': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 2, 'b200tfs_decode_results': 2}, 'concat_device_calls': 0, 'launches': 2, 'result': ['raise', 'KeyError'], 'seen_varints': False, 'stats': [2, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 2, 'b200tfs_decode_results': 2}, 'concat_device_calls': 0, 'launches': 2, 'result': ['raise', 'KeyError'], 'seen_varints': False, 'stats': [2, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 2, 'b200tfs_decode_results': 2, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 2, 'result': ['raise', 'KeyError'], 'seen_varints': True, 'stats': [2, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 2, 'b200tfs_decode_results': 2, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 2, 'result': ['raise', 'KeyError'], 'seen_varints': True, 'stats': [2, 0, 0]},
        ],
    },
    'out_pinned_out_dtypes': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_set_decode_cast': 2}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[['y', ['array', '<f2', [64, 33], '37819bd42f3f', 'out']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_set_decode_cast': 2}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[['y', ['array', '<f2', [64, 33], '37819bd42f3f', 'out']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_cast': 2}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[['y', ['array', '<f2', [64, 33], '37819bd42f3f', 'out']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_cast': 2}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[['y', ['array', '<f2', [64, 33], '37819bd42f3f', 'out']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'out_pinned_shape_mismatch': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 2, 'b200tfs_decode_results': 2}, 'concat_device_calls': 0, 'launches': 2, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [1, 0, 1]},
            {'calls': {'b200tfs_decode_responses_host_async': 2, 'b200tfs_decode_results': 2}, 'concat_device_calls': 0, 'launches': 2, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [1, 0, 1]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 2, 'b200tfs_decode_results': 2, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 2, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [1, 0, 1]},
            {'calls': {'b200tfs_decode_responses_host_async': 2, 'b200tfs_decode_results': 2, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 2, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [1, 0, 1]},
        ],
    },
    'out_pinned_strict': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[['y', ['array', '<f4', [64, 33], '85fc1075c812', 'out']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[['y', ['array', '<f4', [64, 33], '85fc1075c812', 'out']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[['y', ['array', '<f4', [64, 33], '85fc1075c812', 'out']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[['y', ['array', '<f4', [64, 33], '85fc1075c812', 'out']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'out_pinned_truncated': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 2, 'b200tfs_decode_results': 2, 'b200tfs_parse_responses_host': 1}, 'concat_device_calls': 0, 'launches': 3, 'result': ['raise', 'DecodeError'], 'seen_varints': False, 'stats': [0, 0, 2]},
            {'calls': {'b200tfs_decode_responses_host_async': 2, 'b200tfs_decode_results': 2, 'b200tfs_parse_responses_host': 1}, 'concat_device_calls': 0, 'launches': 3, 'result': ['raise', 'DecodeError'], 'seen_varints': False, 'stats': [0, 0, 2]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 2, 'b200tfs_decode_results': 2, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_parse_responses_host': 1}, 'concat_device_calls': 0, 'launches': 3, 'result': ['raise', 'DecodeError'], 'seen_varints': True, 'stats': [0, 0, 2]},
            {'calls': {'b200tfs_decode_responses_host_async': 2, 'b200tfs_decode_results': 2, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_parse_responses_host': 1}, 'concat_device_calls': 0, 'launches': 3, 'result': ['raise', 'DecodeError'], 'seen_varints': True, 'stats': [0, 0, 2]},
        ],
    },
    'out_pinned_two_outputs': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 2, 'b200tfs_decode_results': 2}, 'concat_device_calls': 0, 'launches': 2, 'result': ['ok', [[['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'out']], ['d', ['array', '<f8', [3], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': False, 'stats': [2, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 2, 'b200tfs_decode_results': 2}, 'concat_device_calls': 0, 'launches': 2, 'result': ['ok', [[['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'out']], ['d', ['array', '<f8', [3], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': False, 'stats': [2, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 2, 'b200tfs_decode_results': 2, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 2, 'result': ['ok', [[['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'out']], ['d', ['array', '<f8', [3], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': True, 'stats': [2, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 2, 'b200tfs_decode_results': 2, 'b200tfs_decode_slot_bytes': 1}, 'concat_device_calls': 0, 'launches': 2, 'result': ['ok', [[['scores', ['array', '<f4', [8, 5], '640ba4d3c6af', 'out']], ['d', ['array', '<f8', [3], '7f0639ce5dac', 'view']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': True, 'stats': [2, 0, 0]},
        ],
    },
    'out_pinned_varint': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 2, 'b200tfs_decode_results': 2, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 5, 'result': ['ok', [[['ids', ['array', '<i8', [7], '6984488c7681', 'out']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': True, 'stats': [2, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 2, 'b200tfs_decode_results': 2, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 5, 'result': ['ok', [[['ids', ['array', '<i8', [7], '6984488c7681', 'out']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': True, 'stats': [2, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 2, 'b200tfs_decode_results': 2, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 5, 'result': ['ok', [[['ids', ['array', '<i8', [7], '6984488c7681', 'out']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': True, 'stats': [2, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 2, 'b200tfs_decode_results': 2, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_set_decode_varints': 2}, 'concat_device_calls': 0, 'launches': 5, 'result': ['ok', [[['ids', ['array', '<i8', [7], '6984488c7681', 'out']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': True, 'stats': [2, 0, 0]},
        ],
    },
    'out_pinned_wire': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[['y', ['array', '<f4', [64, 33], '85fc1075c812', 'out']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': False, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[['y', ['array', '<f4', [64, 33], '85fc1075c812', 'out']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': False, 'stats': [1, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[['y', ['array', '<f4', [64, 33], '85fc1075c812', 'out']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': True, 'stats': [1, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 1, 'b200tfs_decode_results': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [[['y', ['array', '<f4', [64, 33], '85fc1075c812', 'out']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': True, 'stats': [1, 0, 0]},
        ],
    },
    'out_pinned_zero_none': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 2, 'b200tfs_decode_results': 2, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 2, 'result': ['ok', [[['y', ['array', '<f4', [0], 'da39a3ee5e6b', 'out']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': False, 'stats': [2, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 2, 'b200tfs_decode_results': 2, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 2, 'result': ['ok', [[['y', ['array', '<f4', [0], 'da39a3ee5e6b', 'out']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': False, 'stats': [2, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 2, 'b200tfs_decode_results': 2, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 2, 'result': ['ok', [[['y', ['array', '<f4', [0], 'da39a3ee5e6b', 'out']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': True, 'stats': [2, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 2, 'b200tfs_decode_results': 2, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 2, 'result': ['ok', [[['y', ['array', '<f4', [0], 'da39a3ee5e6b', 'out']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': True, 'stats': [2, 0, 0]},
        ],
    },
    'out_pinned_zero_run': {
        'cold': [
            {'calls': {'b200tfs_decode_responses_host_async': 2, 'b200tfs_decode_results': 2, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 2, 'result': ['ok', [[['y', ['array', '<f4', [0], 'da39a3ee5e6b', 'out']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': False, 'stats': [2, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 2, 'b200tfs_decode_results': 2, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 2, 'result': ['ok', [[['y', ['array', '<f4', [0], 'da39a3ee5e6b', 'out']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': False, 'stats': [2, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_responses_host_async': 2, 'b200tfs_decode_results': 2, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 2, 'result': ['ok', [[['y', ['array', '<f4', [0], 'da39a3ee5e6b', 'out']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': True, 'stats': [2, 0, 0]},
            {'calls': {'b200tfs_decode_responses_host_async': 2, 'b200tfs_decode_results': 2, 'b200tfs_decode_slot_bytes': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 2, 'result': ['ok', [[['y', ['array', '<f4', [0], 'da39a3ee5e6b', 'out']]], ['spec', 'default', 1, True, '', 'serving_default']]], 'seen_varints': True, 'stats': [2, 0, 0]},
        ],
    },
    'padded_content': {
        'cold': [
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[['c', ['array', '<f4', [16, 5], '0faa8a48c67b', 'fresh']]], [['c', ['array', '<i8', [2, 2], '825a637d87fb', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[['c', ['array', '<f4', [16, 5], '0faa8a48c67b', 'fresh']]], [['c', ['array', '<i8', [2, 2], '825a637d87fb', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[['c', ['array', '<f4', [16, 5], '0faa8a48c67b', 'fresh']]], [['c', ['array', '<i8', [2, 2], '825a637d87fb', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[['c', ['array', '<f4', [16, 5], '0faa8a48c67b', 'fresh']]], [['c', ['array', '<i8', [2, 2], '825a637d87fb', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'padded_dtype_disagrees': {
        'cold': [
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'padded_floats': {
        'cold': [
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['scores', ['array', '<f4', [24, 5], '907117f39572', 'fresh']], ['d', ['array', '<f8', [9], 'ac70ecbf4f0c', 'fresh']]], [['scores', ['array', '<i8', [3, 2], '8d1645f09d1d', 'fresh']], ['d', ['array', '<i8', [3, 1], 'de29d662a270', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['scores', ['array', '<f4', [24, 5], '907117f39572', 'fresh']], ['d', ['array', '<f8', [9], 'ac70ecbf4f0c', 'fresh']]], [['scores', ['array', '<i8', [3, 2], '8d1645f09d1d', 'fresh']], ['d', ['array', '<i8', [3, 1], 'de29d662a270', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['scores', ['array', '<f4', [24, 5], '907117f39572', 'fresh']], ['d', ['array', '<f8', [9], 'ac70ecbf4f0c', 'fresh']]], [['scores', ['array', '<i8', [3, 2], '8d1645f09d1d', 'fresh']], ['d', ['array', '<i8', [3, 1], 'de29d662a270', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['scores', ['array', '<f4', [24, 5], '907117f39572', 'fresh']], ['d', ['array', '<f8', [9], 'ac70ecbf4f0c', 'fresh']]], [['scores', ['array', '<i8', [3, 2], '8d1645f09d1d', 'fresh']], ['d', ['array', '<i8', [3, 1], 'de29d662a270', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'padded_floats_device': {
        'cold': [
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['scores', ['device', '<f4', [24, 5], '907117f39572', 'device']], ['d', ['device', '<f8', [9], 'ac70ecbf4f0c', 'device']]], [['scores', ['array', '<i8', [3, 2], '8d1645f09d1d', 'fresh']], ['d', ['array', '<i8', [3, 1], 'de29d662a270', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['scores', ['device', '<f4', [24, 5], '907117f39572', 'device']], ['d', ['device', '<f8', [9], 'ac70ecbf4f0c', 'device']]], [['scores', ['array', '<i8', [3, 2], '8d1645f09d1d', 'fresh']], ['d', ['array', '<i8', [3, 1], 'de29d662a270', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['scores', ['device', '<f4', [24, 5], '907117f39572', 'device']], ['d', ['device', '<f8', [9], 'ac70ecbf4f0c', 'device']]], [['scores', ['array', '<i8', [3, 2], '8d1645f09d1d', 'fresh']], ['d', ['array', '<i8', [3, 1], 'de29d662a270', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['scores', ['device', '<f4', [24, 5], '907117f39572', 'device']], ['d', ['device', '<f8', [9], 'ac70ecbf4f0c', 'device']]], [['scores', ['array', '<i8', [3, 2], '8d1645f09d1d', 'fresh']], ['d', ['array', '<i8', [3, 1], 'de29d662a270', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'padded_half': {
        'cold': [
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['h', ['array', '<f2', [12], 'd7d38c467a05', 'fresh']], ['f', ['array', '<f4', [10], '978ac77ea8bf', 'fresh']]], [['h', ['array', '<i8', [2, 1], '61434fbc6460', 'fresh']], ['f', ['array', '<i8', [2, 1], '37089f813939', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['h', ['array', '<f2', [12], 'd7d38c467a05', 'fresh']], ['f', ['array', '<f4', [10], '978ac77ea8bf', 'fresh']]], [['h', ['array', '<i8', [2, 1], '61434fbc6460', 'fresh']], ['f', ['array', '<i8', [2, 1], '37089f813939', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['h', ['array', '<f2', [12], 'd7d38c467a05', 'fresh']], ['f', ['array', '<f4', [10], '978ac77ea8bf', 'fresh']]], [['h', ['array', '<i8', [2, 1], '61434fbc6460', 'fresh']], ['f', ['array', '<i8', [2, 1], '37089f813939', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['h', ['array', '<f2', [12], 'd7d38c467a05', 'fresh']], ['f', ['array', '<f4', [10], '978ac77ea8bf', 'fresh']]], [['h', ['array', '<i8', [2, 1], '61434fbc6460', 'fresh']], ['f', ['array', '<i8', [2, 1], '37089f813939', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'padded_half_strict': {
        'cold': [
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 8, 'result': ['ok', [[['h', ['array', '<f2', [12], 'a612ac46cb97', 'fresh']], ['f', ['array', '<f4', [10], '978ac77ea8bf', 'fresh']]], [['h', ['array', '<i8', [2, 1], '61434fbc6460', 'fresh']], ['f', ['array', '<i8', [2, 1], '37089f813939', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 8, 'result': ['ok', [[['h', ['array', '<f2', [12], 'a612ac46cb97', 'fresh']], ['f', ['array', '<f4', [10], '978ac77ea8bf', 'fresh']]], [['h', ['array', '<i8', [2, 1], '61434fbc6460', 'fresh']], ['f', ['array', '<i8', [2, 1], '37089f813939', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 8, 'result': ['ok', [[['h', ['array', '<f2', [12], 'a612ac46cb97', 'fresh']], ['f', ['array', '<f4', [10], '978ac77ea8bf', 'fresh']]], [['h', ['array', '<i8', [2, 1], '61434fbc6460', 'fresh']], ['f', ['array', '<i8', [2, 1], '37089f813939', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 8, 'result': ['ok', [[['h', ['array', '<f2', [12], 'a612ac46cb97', 'fresh']], ['f', ['array', '<f4', [10], '978ac77ea8bf', 'fresh']]], [['h', ['array', '<i8', [2, 1], '61434fbc6460', 'fresh']], ['f', ['array', '<i8', [2, 1], '37089f813939', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'padded_keys': {
        'cold': [
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['d', ['array', '<f8', [4, 1], '29fc26da5c1c', 'fresh']], ['classes', ['array', '<i8', [10, 5], 'db935af57046', 'fresh']]], [['d', ['array', '<i8', [2, 2], '8a9fb03e4ef2', 'fresh']], ['classes', ['array', '<i8', [2, 2], '4a72c2d2a443', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['d', ['array', '<f8', [4, 1], '29fc26da5c1c', 'fresh']], ['classes', ['array', '<i8', [10, 5], 'db935af57046', 'fresh']]], [['d', ['array', '<i8', [2, 2], '8a9fb03e4ef2', 'fresh']], ['classes', ['array', '<i8', [2, 2], '4a72c2d2a443', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['d', ['array', '<f8', [4, 1], '29fc26da5c1c', 'fresh']], ['classes', ['array', '<i8', [10, 5], 'db935af57046', 'fresh']]], [['d', ['array', '<i8', [2, 2], '8a9fb03e4ef2', 'fresh']], ['classes', ['array', '<i8', [2, 2], '4a72c2d2a443', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['d', ['array', '<f8', [4, 1], '29fc26da5c1c', 'fresh']], ['classes', ['array', '<i8', [10, 5], 'db935af57046', 'fresh']]], [['d', ['array', '<i8', [2, 2], '8a9fb03e4ef2', 'fresh']], ['classes', ['array', '<i8', [2, 2], '4a72c2d2a443', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'padded_many': {
        'cold': [
            {'calls': {'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[['o0', ['array', '<f4', [10], '978ac77ea8bf', 'fresh']], ['o1', ['array', '<f4', [10], '9bd4809dc080', 'fresh']], ['o2', ['array', '<f4', [10], '603b11843256', 'fresh']], ['o3', ['array', '<f4', [10], '12388578a29e', 'fresh']], ['o4', ['array', '<f4', [10], '50493d3f1088', 'fresh']], ['o5', ['array', '<f4', [10], '159f97f92d1a', 'fresh']], ['o6', ['array', '<f4', [10], '4d18a2bb7161', 'fresh']], ['o7', ['array', '<f4', [10], '361fa970ef6e', 'fresh']], ['o8', ['array', '<f4', [10], '2b195ee6133a', 'fresh']]], [['o0', ['array', '<i8', [2, 1], '37089f813939', 'fresh']], ['o1', ['array', '<i8', [2, 1], '37089f813939', 'fresh']], ['o2', ['array', '<i8', [2, 1], '37089f813939', 'fresh']], ['o3', ['array', '<i8', [2, 1], '37089f813939', 'fresh']], ['o4', ['array', '<i8', [2, 1], '37089f813939', 'fresh']], ['o5', ['array', '<i8', [2, 1], '37089f813939', 'fresh']], ['o6', ['array', '<i8', [2, 1], '37089f813939', 'fresh']], ['o7', ['array', '<i8', [2, 1], '37089f813939', 'fresh']], ['o8', ['array', '<i8', [2, 1], '37089f813939', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[['o0', ['array', '<f4', [10], '978ac77ea8bf', 'fresh']], ['o1', ['array', '<f4', [10], '9bd4809dc080', 'fresh']], ['o2', ['array', '<f4', [10], '603b11843256', 'fresh']], ['o3', ['array', '<f4', [10], '12388578a29e', 'fresh']], ['o4', ['array', '<f4', [10], '50493d3f1088', 'fresh']], ['o5', ['array', '<f4', [10], '159f97f92d1a', 'fresh']], ['o6', ['array', '<f4', [10], '4d18a2bb7161', 'fresh']], ['o7', ['array', '<f4', [10], '361fa970ef6e', 'fresh']], ['o8', ['array', '<f4', [10], '2b195ee6133a', 'fresh']]], [['o0', ['array', '<i8', [2, 1], '37089f813939', 'fresh']], ['o1', ['array', '<i8', [2, 1], '37089f813939', 'fresh']], ['o2', ['array', '<i8', [2, 1], '37089f813939', 'fresh']], ['o3', ['array', '<i8', [2, 1], '37089f813939', 'fresh']], ['o4', ['array', '<i8', [2, 1], '37089f813939', 'fresh']], ['o5', ['array', '<i8', [2, 1], '37089f813939', 'fresh']], ['o6', ['array', '<i8', [2, 1], '37089f813939', 'fresh']], ['o7', ['array', '<i8', [2, 1], '37089f813939', 'fresh']], ['o8', ['array', '<i8', [2, 1], '37089f813939', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[['o0', ['array', '<f4', [10], '978ac77ea8bf', 'fresh']], ['o1', ['array', '<f4', [10], '9bd4809dc080', 'fresh']], ['o2', ['array', '<f4', [10], '603b11843256', 'fresh']], ['o3', ['array', '<f4', [10], '12388578a29e', 'fresh']], ['o4', ['array', '<f4', [10], '50493d3f1088', 'fresh']], ['o5', ['array', '<f4', [10], '159f97f92d1a', 'fresh']], ['o6', ['array', '<f4', [10], '4d18a2bb7161', 'fresh']], ['o7', ['array', '<f4', [10], '361fa970ef6e', 'fresh']], ['o8', ['array', '<f4', [10], '2b195ee6133a', 'fresh']]], [['o0', ['array', '<i8', [2, 1], '37089f813939', 'fresh']], ['o1', ['array', '<i8', [2, 1], '37089f813939', 'fresh']], ['o2', ['array', '<i8', [2, 1], '37089f813939', 'fresh']], ['o3', ['array', '<i8', [2, 1], '37089f813939', 'fresh']], ['o4', ['array', '<i8', [2, 1], '37089f813939', 'fresh']], ['o5', ['array', '<i8', [2, 1], '37089f813939', 'fresh']], ['o6', ['array', '<i8', [2, 1], '37089f813939', 'fresh']], ['o7', ['array', '<i8', [2, 1], '37089f813939', 'fresh']], ['o8', ['array', '<i8', [2, 1], '37089f813939', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[['o0', ['array', '<f4', [10], '978ac77ea8bf', 'fresh']], ['o1', ['array', '<f4', [10], '9bd4809dc080', 'fresh']], ['o2', ['array', '<f4', [10], '603b11843256', 'fresh']], ['o3', ['array', '<f4', [10], '12388578a29e', 'fresh']], ['o4', ['array', '<f4', [10], '50493d3f1088', 'fresh']], ['o5', ['array', '<f4', [10], '159f97f92d1a', 'fresh']], ['o6', ['array', '<f4', [10], '4d18a2bb7161', 'fresh']], ['o7', ['array', '<f4', [10], '361fa970ef6e', 'fresh']], ['o8', ['array', '<f4', [10], '2b195ee6133a', 'fresh']]], [['o0', ['array', '<i8', [2, 1], '37089f813939', 'fresh']], ['o1', ['array', '<i8', [2, 1], '37089f813939', 'fresh']], ['o2', ['array', '<i8', [2, 1], '37089f813939', 'fresh']], ['o3', ['array', '<i8', [2, 1], '37089f813939', 'fresh']], ['o4', ['array', '<i8', [2, 1], '37089f813939', 'fresh']], ['o5', ['array', '<i8', [2, 1], '37089f813939', 'fresh']], ['o6', ['array', '<i8', [2, 1], '37089f813939', 'fresh']], ['o7', ['array', '<i8', [2, 1], '37089f813939', 'fresh']], ['o8', ['array', '<i8', [2, 1], '37089f813939', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'padded_mixed': {
        'cold': [
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 3, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['classes', ['array', '<i8', [10, 5], 'db935af57046', 'fresh']], ['scores', ['array', '<f4', [10, 5], '61c2992f9901', 'fresh']], ['d', ['array', '<f8', [4, 1], '29fc26da5c1c', 'fresh']]], [['classes', ['array', '<i8', [2, 2], '4a72c2d2a443', 'fresh']], ['scores', ['array', '<i8', [2, 2], '4a72c2d2a443', 'fresh']], ['d', ['array', '<i8', [2, 2], '8a9fb03e4ef2', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 3, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['classes', ['array', '<i8', [10, 5], 'db935af57046', 'fresh']], ['scores', ['array', '<f4', [10, 5], '61c2992f9901', 'fresh']], ['d', ['array', '<f8', [4, 1], '29fc26da5c1c', 'fresh']]], [['classes', ['array', '<i8', [2, 2], '4a72c2d2a443', 'fresh']], ['scores', ['array', '<i8', [2, 2], '4a72c2d2a443', 'fresh']], ['d', ['array', '<i8', [2, 2], '8a9fb03e4ef2', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 3, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['classes', ['array', '<i8', [10, 5], 'db935af57046', 'fresh']], ['scores', ['array', '<f4', [10, 5], '61c2992f9901', 'fresh']], ['d', ['array', '<f8', [4, 1], '29fc26da5c1c', 'fresh']]], [['classes', ['array', '<i8', [2, 2], '4a72c2d2a443', 'fresh']], ['scores', ['array', '<i8', [2, 2], '4a72c2d2a443', 'fresh']], ['d', ['array', '<i8', [2, 2], '8a9fb03e4ef2', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 3, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['classes', ['array', '<i8', [10, 5], 'db935af57046', 'fresh']], ['scores', ['array', '<f4', [10, 5], '61c2992f9901', 'fresh']], ['d', ['array', '<f8', [4, 1], '29fc26da5c1c', 'fresh']]], [['classes', ['array', '<i8', [2, 2], '4a72c2d2a443', 'fresh']], ['scores', ['array', '<i8', [2, 2], '4a72c2d2a443', 'fresh']], ['d', ['array', '<i8', [2, 2], '8a9fb03e4ef2', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'padded_mixed_device': {
        'cold': [
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['classes', ['device', '<i8', [10, 5], 'db935af57046', 'device']], ['scores', ['device', '<f4', [10, 5], '61c2992f9901', 'device']], ['d', ['device', '<f8', [4, 1], '29fc26da5c1c', 'device']]], [['classes', ['array', '<i8', [2, 2], '4a72c2d2a443', 'fresh']], ['scores', ['array', '<i8', [2, 2], '4a72c2d2a443', 'fresh']], ['d', ['array', '<i8', [2, 2], '8a9fb03e4ef2', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['classes', ['device', '<i8', [10, 5], 'db935af57046', 'device']], ['scores', ['device', '<f4', [10, 5], '61c2992f9901', 'device']], ['d', ['device', '<f8', [4, 1], '29fc26da5c1c', 'device']]], [['classes', ['array', '<i8', [2, 2], '4a72c2d2a443', 'fresh']], ['scores', ['array', '<i8', [2, 2], '4a72c2d2a443', 'fresh']], ['d', ['array', '<i8', [2, 2], '8a9fb03e4ef2', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['classes', ['device', '<i8', [10, 5], 'db935af57046', 'device']], ['scores', ['device', '<f4', [10, 5], '61c2992f9901', 'device']], ['d', ['device', '<f8', [4, 1], '29fc26da5c1c', 'device']]], [['classes', ['array', '<i8', [2, 2], '4a72c2d2a443', 'fresh']], ['scores', ['array', '<i8', [2, 2], '4a72c2d2a443', 'fresh']], ['d', ['array', '<i8', [2, 2], '8a9fb03e4ef2', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['classes', ['device', '<i8', [10, 5], 'db935af57046', 'device']], ['scores', ['device', '<f4', [10, 5], '61c2992f9901', 'device']], ['d', ['device', '<f8', [4, 1], '29fc26da5c1c', 'device']]], [['classes', ['array', '<i8', [2, 2], '4a72c2d2a443', 'fresh']], ['scores', ['array', '<i8', [2, 2], '4a72c2d2a443', 'fresh']], ['d', ['array', '<i8', [2, 2], '8a9fb03e4ef2', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'padded_mixed_strict': {
        'cold': [
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 3, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['classes', ['array', '<i8', [10, 5], 'db935af57046', 'fresh']], ['scores', ['array', '<f4', [10, 5], '61c2992f9901', 'fresh']], ['d', ['array', '<f8', [4, 1], '29fc26da5c1c', 'fresh']]], [['classes', ['array', '<i8', [2, 2], '4a72c2d2a443', 'fresh']], ['scores', ['array', '<i8', [2, 2], '4a72c2d2a443', 'fresh']], ['d', ['array', '<i8', [2, 2], '8a9fb03e4ef2', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 3, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['classes', ['array', '<i8', [10, 5], 'db935af57046', 'fresh']], ['scores', ['array', '<f4', [10, 5], '61c2992f9901', 'fresh']], ['d', ['array', '<f8', [4, 1], '29fc26da5c1c', 'fresh']]], [['classes', ['array', '<i8', [2, 2], '4a72c2d2a443', 'fresh']], ['scores', ['array', '<i8', [2, 2], '4a72c2d2a443', 'fresh']], ['d', ['array', '<i8', [2, 2], '8a9fb03e4ef2', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 3, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['classes', ['array', '<i8', [10, 5], 'db935af57046', 'fresh']], ['scores', ['array', '<f4', [10, 5], '61c2992f9901', 'fresh']], ['d', ['array', '<f8', [4, 1], '29fc26da5c1c', 'fresh']]], [['classes', ['array', '<i8', [2, 2], '4a72c2d2a443', 'fresh']], ['scores', ['array', '<i8', [2, 2], '4a72c2d2a443', 'fresh']], ['d', ['array', '<i8', [2, 2], '8a9fb03e4ef2', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 3, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['classes', ['array', '<i8', [10, 5], 'db935af57046', 'fresh']], ['scores', ['array', '<f4', [10, 5], '61c2992f9901', 'fresh']], ['d', ['array', '<f8', [4, 1], '29fc26da5c1c', 'fresh']]], [['classes', ['array', '<i8', [2, 2], '4a72c2d2a443', 'fresh']], ['scores', ['array', '<i8', [2, 2], '4a72c2d2a443', 'fresh']], ['d', ['array', '<i8', [2, 2], '8a9fb03e4ef2', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'padded_narrow': {
        'cold': [
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 3, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1, 'b200tfs_set_decode_cast': 2}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['f', ['array', '<f2', [60, 7], '1ef8d77aafaa', 'fresh']], ['g', ['array', '<f2', [198], '01c90ef1748f', 'fresh']], ['ids', ['array', '<i8', [100], '4b0fdc7daed0', 'fresh']]], [['f', ['array', '<i8', [2, 2], 'e64d738ca8ff', 'fresh']], ['g', ['array', '<i8', [2, 1], '706e0b8d481d', 'fresh']], ['ids', ['array', '<i8', [2, 1], '5835af0410d0', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 3, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1, 'b200tfs_set_decode_cast': 2}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['f', ['array', '<f2', [60, 7], '1ef8d77aafaa', 'fresh']], ['g', ['array', '<f2', [198], '01c90ef1748f', 'fresh']], ['ids', ['array', '<i8', [100], '4b0fdc7daed0', 'fresh']]], [['f', ['array', '<i8', [2, 2], 'e64d738ca8ff', 'fresh']], ['g', ['array', '<i8', [2, 1], '706e0b8d481d', 'fresh']], ['ids', ['array', '<i8', [2, 1], '5835af0410d0', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 3, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1, 'b200tfs_set_decode_cast': 2}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['f', ['array', '<f2', [60, 7], '1ef8d77aafaa', 'fresh']], ['g', ['array', '<f2', [198], '01c90ef1748f', 'fresh']], ['ids', ['array', '<i8', [100], '4b0fdc7daed0', 'fresh']]], [['f', ['array', '<i8', [2, 2], 'e64d738ca8ff', 'fresh']], ['g', ['array', '<i8', [2, 1], '706e0b8d481d', 'fresh']], ['ids', ['array', '<i8', [2, 1], '5835af0410d0', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 3, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1, 'b200tfs_set_decode_cast': 2}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['f', ['array', '<f2', [60, 7], '1ef8d77aafaa', 'fresh']], ['g', ['array', '<f2', [198], '01c90ef1748f', 'fresh']], ['ids', ['array', '<i8', [100], '4b0fdc7daed0', 'fresh']]], [['f', ['array', '<i8', [2, 2], 'e64d738ca8ff', 'fresh']], ['g', ['array', '<i8', [2, 1], '706e0b8d481d', 'fresh']], ['ids', ['array', '<i8', [2, 1], '5835af0410d0', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'padded_narrow_partial': {
        'cold': [
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 10, 'result': ['ok', [[['f', ['array', '<f2', [60, 7], '1ef8d77aafaa', 'fresh']], ['g', ['array', '<f4', [198], 'ea065140f6b0', 'fresh']], ['ids', ['array', '<i8', [100], '4b0fdc7daed0', 'fresh']]], [['f', ['array', '<i8', [2, 2], 'e64d738ca8ff', 'fresh']], ['g', ['array', '<i8', [2, 1], '706e0b8d481d', 'fresh']], ['ids', ['array', '<i8', [2, 1], '5835af0410d0', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 10, 'result': ['ok', [[['f', ['array', '<f2', [60, 7], '1ef8d77aafaa', 'fresh']], ['g', ['array', '<f4', [198], 'ea065140f6b0', 'fresh']], ['ids', ['array', '<i8', [100], '4b0fdc7daed0', 'fresh']]], [['f', ['array', '<i8', [2, 2], 'e64d738ca8ff', 'fresh']], ['g', ['array', '<i8', [2, 1], '706e0b8d481d', 'fresh']], ['ids', ['array', '<i8', [2, 1], '5835af0410d0', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 10, 'result': ['ok', [[['f', ['array', '<f2', [60, 7], '1ef8d77aafaa', 'fresh']], ['g', ['array', '<f4', [198], 'ea065140f6b0', 'fresh']], ['ids', ['array', '<i8', [100], '4b0fdc7daed0', 'fresh']]], [['f', ['array', '<i8', [2, 2], 'e64d738ca8ff', 'fresh']], ['g', ['array', '<i8', [2, 1], '706e0b8d481d', 'fresh']], ['ids', ['array', '<i8', [2, 1], '5835af0410d0', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 10, 'result': ['ok', [[['f', ['array', '<f2', [60, 7], '1ef8d77aafaa', 'fresh']], ['g', ['array', '<f4', [198], 'ea065140f6b0', 'fresh']], ['ids', ['array', '<i8', [100], '4b0fdc7daed0', 'fresh']]], [['f', ['array', '<i8', [2, 2], 'e64d738ca8ff', 'fresh']], ['g', ['array', '<i8', [2, 1], '706e0b8d481d', 'fresh']], ['ids', ['array', '<i8', [2, 1], '5835af0410d0', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'padded_narrow_strict': {
        'cold': [
            {'calls': {'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 8, 'result': ['ok', [[['f', ['array', '<f2', [60, 7], '1ef8d77aafaa', 'fresh']], ['g', ['array', '<f2', [198], '01c90ef1748f', 'fresh']], ['ids', ['array', '<i8', [100], '4b0fdc7daed0', 'fresh']]], [['f', ['array', '<i8', [2, 2], 'e64d738ca8ff', 'fresh']], ['g', ['array', '<i8', [2, 1], '706e0b8d481d', 'fresh']], ['ids', ['array', '<i8', [2, 1], '5835af0410d0', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 8, 'result': ['ok', [[['f', ['array', '<f2', [60, 7], '1ef8d77aafaa', 'fresh']], ['g', ['array', '<f2', [198], '01c90ef1748f', 'fresh']], ['ids', ['array', '<i8', [100], '4b0fdc7daed0', 'fresh']]], [['f', ['array', '<i8', [2, 2], 'e64d738ca8ff', 'fresh']], ['g', ['array', '<i8', [2, 1], '706e0b8d481d', 'fresh']], ['ids', ['array', '<i8', [2, 1], '5835af0410d0', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 8, 'result': ['ok', [[['f', ['array', '<f2', [60, 7], '1ef8d77aafaa', 'fresh']], ['g', ['array', '<f2', [198], '01c90ef1748f', 'fresh']], ['ids', ['array', '<i8', [100], '4b0fdc7daed0', 'fresh']]], [['f', ['array', '<i8', [2, 2], 'e64d738ca8ff', 'fresh']], ['g', ['array', '<i8', [2, 1], '706e0b8d481d', 'fresh']], ['ids', ['array', '<i8', [2, 1], '5835af0410d0', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 8, 'result': ['ok', [[['f', ['array', '<f2', [60, 7], '1ef8d77aafaa', 'fresh']], ['g', ['array', '<f2', [198], '01c90ef1748f', 'fresh']], ['ids', ['array', '<i8', [100], '4b0fdc7daed0', 'fresh']]], [['f', ['array', '<i8', [2, 2], 'e64d738ca8ff', 'fresh']], ['g', ['array', '<i8', [2, 1], '706e0b8d481d', 'fresh']], ['ids', ['array', '<i8', [2, 1], '5835af0410d0', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'padded_out_device': {
        'cold': [
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_h2d': 3, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['scores', ['device', '<f4', [16, 5], '9808d3628a01', 'out']], ['d', ['device', '<f8', [6], '9f573d120c9b', 'out']]], [['scores', ['array', '<i8', [2, 2], '825a637d87fb', 'fresh']], ['d', ['array', '<i8', [2, 1], '7590cbf3642e', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_h2d': 3, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['scores', ['device', '<f4', [16, 5], '9808d3628a01', 'out']], ['d', ['device', '<f8', [6], '9f573d120c9b', 'out']]], [['scores', ['array', '<i8', [2, 2], '825a637d87fb', 'fresh']], ['d', ['array', '<i8', [2, 1], '7590cbf3642e', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_h2d': 3, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['scores', ['device', '<f4', [16, 5], '9808d3628a01', 'out']], ['d', ['device', '<f8', [6], '9f573d120c9b', 'out']]], [['scores', ['array', '<i8', [2, 2], '825a637d87fb', 'fresh']], ['d', ['array', '<i8', [2, 1], '7590cbf3642e', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_h2d': 3, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['scores', ['device', '<f4', [16, 5], '9808d3628a01', 'out']], ['d', ['device', '<f8', [6], '9f573d120c9b', 'out']]], [['scores', ['array', '<i8', [2, 2], '825a637d87fb', 'fresh']], ['d', ['array', '<i8', [2, 1], '7590cbf3642e', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'padded_out_device_mismatch': {
        'cold': [
            {'calls': {'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 0, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 0, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 0, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 0, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'padded_out_mismatch': {
        'cold': [
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 0, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 0, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 0, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 0, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'padded_out_numpy': {
        'cold': [
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['scores', ['array', '<f4', [16, 5], '9808d3628a01', 'out']], ['d', ['array', '<f8', [6], '9f573d120c9b', 'fresh']]], [['scores', ['array', '<i8', [2, 2], '825a637d87fb', 'fresh']], ['d', ['array', '<i8', [2, 1], '7590cbf3642e', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['scores', ['array', '<f4', [16, 5], '9808d3628a01', 'out']], ['d', ['array', '<f8', [6], '9f573d120c9b', 'fresh']]], [['scores', ['array', '<i8', [2, 2], '825a637d87fb', 'fresh']], ['d', ['array', '<i8', [2, 1], '7590cbf3642e', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['scores', ['array', '<f4', [16, 5], '9808d3628a01', 'out']], ['d', ['array', '<f8', [6], '9f573d120c9b', 'fresh']]], [['scores', ['array', '<i8', [2, 2], '825a637d87fb', 'fresh']], ['d', ['array', '<i8', [2, 1], '7590cbf3642e', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['scores', ['array', '<f4', [16, 5], '9808d3628a01', 'out']], ['d', ['array', '<f8', [6], '9f573d120c9b', 'fresh']]], [['scores', ['array', '<i8', [2, 2], '825a637d87fb', 'fresh']], ['d', ['array', '<i8', [2, 1], '7590cbf3642e', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'padded_out_strings_mismatch': {
        'cold': [
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 12, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 12, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 12, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 12, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'padded_out_unaligned': {
        'cold': [
            {'calls': {'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[['scores', ['array', '<f4', [16, 5], '9808d3628a01', 'fresh']], ['d', ['array', '<f8', [6], '9f573d120c9b', 'fresh']]], [['scores', ['array', '<i8', [2, 2], '825a637d87fb', 'fresh']], ['d', ['array', '<i8', [2, 1], '7590cbf3642e', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[['scores', ['array', '<f4', [16, 5], '9808d3628a01', 'fresh']], ['d', ['array', '<f8', [6], '9f573d120c9b', 'fresh']]], [['scores', ['array', '<i8', [2, 2], '825a637d87fb', 'fresh']], ['d', ['array', '<i8', [2, 1], '7590cbf3642e', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[['scores', ['array', '<f4', [16, 5], '9808d3628a01', 'fresh']], ['d', ['array', '<f8', [6], '9f573d120c9b', 'fresh']]], [['scores', ['array', '<i8', [2, 2], '825a637d87fb', 'fresh']], ['d', ['array', '<i8', [2, 1], '7590cbf3642e', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['ok', [[['scores', ['array', '<f4', [16, 5], '9808d3628a01', 'fresh']], ['d', ['array', '<f8', [6], '9f573d120c9b', 'fresh']]], [['scores', ['array', '<i8', [2, 2], '825a637d87fb', 'fresh']], ['d', ['array', '<i8', [2, 1], '7590cbf3642e', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'padded_pad': {
        'cold': [
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['p', ['array', '<f4', [12], 'bb69489226a6', 'fresh']], ['z', ['array', '<f4', [8], 'de8a847bff8c', 'fresh']]], [['p', ['array', '<i8', [2, 1], '61434fbc6460', 'fresh']], ['z', ['array', '<i8', [2, 1], 'a385649cbb41', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['p', ['array', '<f4', [12], 'bb69489226a6', 'fresh']], ['z', ['array', '<f4', [8], 'de8a847bff8c', 'fresh']]], [['p', ['array', '<i8', [2, 1], '61434fbc6460', 'fresh']], ['z', ['array', '<i8', [2, 1], 'a385649cbb41', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['p', ['array', '<f4', [12], 'bb69489226a6', 'fresh']], ['z', ['array', '<f4', [8], 'de8a847bff8c', 'fresh']]], [['p', ['array', '<i8', [2, 1], '61434fbc6460', 'fresh']], ['z', ['array', '<i8', [2, 1], 'a385649cbb41', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['p', ['array', '<f4', [12], 'bb69489226a6', 'fresh']], ['z', ['array', '<f4', [8], 'de8a847bff8c', 'fresh']]], [['p', ['array', '<i8', [2, 1], '61434fbc6460', 'fresh']], ['z', ['array', '<i8', [2, 1], 'a385649cbb41', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'padded_pad_to': {
        'cold': [
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['scores', ['array', '<f4', [13, 9], '301b6605a03b', 'fresh']], ['d', ['array', '<f8', [8], '1744000061fe', 'fresh']]], [['scores', ['array', '<i8', [3, 2], 'b7c568c51e44', 'fresh']], ['d', ['array', '<i8', [3, 1], '46970c330957', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['scores', ['array', '<f4', [13, 9], '301b6605a03b', 'fresh']], ['d', ['array', '<f8', [8], '1744000061fe', 'fresh']]], [['scores', ['array', '<i8', [3, 2], 'b7c568c51e44', 'fresh']], ['d', ['array', '<i8', [3, 1], '46970c330957', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['scores', ['array', '<f4', [13, 9], '301b6605a03b', 'fresh']], ['d', ['array', '<f8', [8], '1744000061fe', 'fresh']]], [['scores', ['array', '<i8', [3, 2], 'b7c568c51e44', 'fresh']], ['d', ['array', '<i8', [3, 1], '46970c330957', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['scores', ['array', '<f4', [13, 9], '301b6605a03b', 'fresh']], ['d', ['array', '<f8', [8], '1744000061fe', 'fresh']]], [['scores', ['array', '<i8', [3, 2], 'b7c568c51e44', 'fresh']], ['d', ['array', '<i8', [3, 1], '46970c330957', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'padded_pad_to_rank': {
        'cold': [
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'padded_pad_to_small': {
        'cold': [
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 3, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 3}, 'concat_device_calls': 0, 'launches': 6, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 3, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 3}, 'concat_device_calls': 0, 'launches': 6, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 3, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 3}, 'concat_device_calls': 0, 'launches': 6, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 3, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 3}, 'concat_device_calls': 0, 'launches': 6, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'padded_pad_value': {
        'cold': [
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['scores', ['array', '<f4', [13, 7], '1cbc08700a7e', 'fresh']], ['d', ['array', '<f8', [8], '1744000061fe', 'fresh']]], [['scores', ['array', '<i8', [3, 2], 'b7c568c51e44', 'fresh']], ['d', ['array', '<i8', [3, 1], '46970c330957', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['scores', ['array', '<f4', [13, 7], '1cbc08700a7e', 'fresh']], ['d', ['array', '<f8', [8], '1744000061fe', 'fresh']]], [['scores', ['array', '<i8', [3, 2], 'b7c568c51e44', 'fresh']], ['d', ['array', '<i8', [3, 1], '46970c330957', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['scores', ['array', '<f4', [13, 7], '1cbc08700a7e', 'fresh']], ['d', ['array', '<f8', [8], '1744000061fe', 'fresh']]], [['scores', ['array', '<i8', [3, 2], 'b7c568c51e44', 'fresh']], ['d', ['array', '<i8', [3, 1], '46970c330957', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['scores', ['array', '<f4', [13, 7], '1cbc08700a7e', 'fresh']], ['d', ['array', '<f8', [8], '1744000061fe', 'fresh']]], [['scores', ['array', '<i8', [3, 2], 'b7c568c51e44', 'fresh']], ['d', ['array', '<i8', [3, 1], '46970c330957', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'padded_pad_value_bad': {
        'cold': [
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'padded_ragged': {
        'cold': [
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['scores', ['array', '<f4', [13, 7], 'c3e1f8c53e49', 'fresh']], ['d', ['array', '<f8', [8], '1744000061fe', 'fresh']]], [['scores', ['array', '<i8', [3, 2], 'b7c568c51e44', 'fresh']], ['d', ['array', '<i8', [3, 1], '46970c330957', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['scores', ['array', '<f4', [13, 7], 'c3e1f8c53e49', 'fresh']], ['d', ['array', '<f8', [8], '1744000061fe', 'fresh']]], [['scores', ['array', '<i8', [3, 2], 'b7c568c51e44', 'fresh']], ['d', ['array', '<i8', [3, 1], '46970c330957', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['scores', ['array', '<f4', [13, 7], 'c3e1f8c53e49', 'fresh']], ['d', ['array', '<f8', [8], '1744000061fe', 'fresh']]], [['scores', ['array', '<i8', [3, 2], 'b7c568c51e44', 'fresh']], ['d', ['array', '<i8', [3, 1], '46970c330957', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 2, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['scores', ['array', '<f4', [13, 7], 'c3e1f8c53e49', 'fresh']], ['d', ['array', '<f8', [8], '1744000061fe', 'fresh']]], [['scores', ['array', '<i8', [3, 2], 'b7c568c51e44', 'fresh']], ['d', ['array', '<i8', [3, 1], '46970c330957', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'padded_ragged_device': {
        'cold': [
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['scores', ['device', '<f4', [13, 7], 'c3e1f8c53e49', 'device']], ['d', ['device', '<f8', [8], '1744000061fe', 'device']]], [['scores', ['array', '<i8', [3, 2], 'b7c568c51e44', 'fresh']], ['d', ['array', '<i8', [3, 1], '46970c330957', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['scores', ['device', '<f4', [13, 7], 'c3e1f8c53e49', 'device']], ['d', ['device', '<f8', [8], '1744000061fe', 'device']]], [['scores', ['array', '<i8', [3, 2], 'b7c568c51e44', 'fresh']], ['d', ['array', '<i8', [3, 1], '46970c330957', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['scores', ['device', '<f4', [13, 7], 'c3e1f8c53e49', 'device']], ['d', ['device', '<f8', [8], '1744000061fe', 'device']]], [['scores', ['array', '<i8', [3, 2], 'b7c568c51e44', 'fresh']], ['d', ['array', '<i8', [3, 1], '46970c330957', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['scores', ['device', '<f4', [13, 7], 'c3e1f8c53e49', 'device']], ['d', ['device', '<f8', [8], '1744000061fe', 'device']]], [['scores', ['array', '<i8', [3, 2], 'b7c568c51e44', 'fresh']], ['d', ['array', '<i8', [3, 1], '46970c330957', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'padded_rank0': {
        'cold': [
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 4, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'padded_strings': {
        'cold': [
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 12, 'result': ['ok', [[['a', ['array', '<f4', [8], '7e0c4ddcde8e', 'fresh']], ['ids', ['array', '<i8', [12], 'b1e1d436fa4c', 'fresh']], ['m', ['array', '|b1', [10], '86cd1efe8a37', 'fresh']], ['s', ['array', '<U3', [4], '45a441b904fa', 'fresh']]], [['a', ['array', '<i8', [2, 1], 'a385649cbb41', 'fresh']], ['ids', ['array', '<i8', [2, 1], '61434fbc6460', 'fresh']], ['m', ['array', '<i8', [2, 1], '37089f813939', 'fresh']], ['s', ['array', '<i8', [2, 1], '21fdd1ec71ba', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 12, 'result': ['ok', [[['a', ['array', '<f4', [8], '7e0c4ddcde8e', 'fresh']], ['ids', ['array', '<i8', [12], 'b1e1d436fa4c', 'fresh']], ['m', ['array', '|b1', [10], '86cd1efe8a37', 'fresh']], ['s', ['array', '<U3', [4], '45a441b904fa', 'fresh']]], [['a', ['array', '<i8', [2, 1], 'a385649cbb41', 'fresh']], ['ids', ['array', '<i8', [2, 1], '61434fbc6460', 'fresh']], ['m', ['array', '<i8', [2, 1], '37089f813939', 'fresh']], ['s', ['array', '<i8', [2, 1], '21fdd1ec71ba', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 12, 'result': ['ok', [[['a', ['array', '<f4', [8], '7e0c4ddcde8e', 'fresh']], ['ids', ['array', '<i8', [12], 'b1e1d436fa4c', 'fresh']], ['m', ['array', '|b1', [10], '86cd1efe8a37', 'fresh']], ['s', ['array', '<U3', [4], '45a441b904fa', 'fresh']]], [['a', ['array', '<i8', [2, 1], 'a385649cbb41', 'fresh']], ['ids', ['array', '<i8', [2, 1], '61434fbc6460', 'fresh']], ['m', ['array', '<i8', [2, 1], '37089f813939', 'fresh']], ['s', ['array', '<i8', [2, 1], '21fdd1ec71ba', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 12, 'result': ['ok', [[['a', ['array', '<f4', [8], '7e0c4ddcde8e', 'fresh']], ['ids', ['array', '<i8', [12], 'b1e1d436fa4c', 'fresh']], ['m', ['array', '|b1', [10], '86cd1efe8a37', 'fresh']], ['s', ['array', '<U3', [4], '45a441b904fa', 'fresh']]], [['a', ['array', '<i8', [2, 1], 'a385649cbb41', 'fresh']], ['ids', ['array', '<i8', [2, 1], '61434fbc6460', 'fresh']], ['m', ['array', '<i8', [2, 1], '37089f813939', 'fresh']], ['s', ['array', '<i8', [2, 1], '21fdd1ec71ba', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'padded_strings_device': {
        'cold': [
            {'calls': {'b200tfs_memcpy_h2d': 3, 'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 12, 'result': ['raise', 'TypeError'], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_memcpy_h2d': 3, 'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 12, 'result': ['raise', 'TypeError'], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_memcpy_h2d': 3, 'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 12, 'result': ['raise', 'TypeError'], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_memcpy_h2d': 3, 'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 12, 'result': ['raise', 'TypeError'], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'padded_truncated_first': {
        'cold': [
            {'calls': {'b200tfs_parse_responses_host': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'DecodeError'], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_parse_responses_host': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'DecodeError'], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_parse_responses_host': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'DecodeError'], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_parse_responses_host': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'DecodeError'], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'padded_truncated_second': {
        'cold': [
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['raise', 'DecodeError'], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['raise', 'DecodeError'], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['raise', 'DecodeError'], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['raise', 'DecodeError'], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'padded_varint': {
        'cold': [
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 3, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['ids', ['array', '<i8', [6, 7], 'b1151a4651e4', 'fresh']], ['mask', ['array', '|b1', [18], '80e4d63ffc4a', 'fresh']], ['small', ['array', '<i4', [10], 'eee5b0893685', 'fresh']]], [['ids', ['array', '<i8', [2, 2], '1e1a11cce185', 'fresh']], ['mask', ['array', '<i8', [2, 1], '23b8f6f42560', 'fresh']], ['small', ['array', '<i8', [2, 1], '37089f813939', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 3, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['ids', ['array', '<i8', [6, 7], 'b1151a4651e4', 'fresh']], ['mask', ['array', '|b1', [18], '80e4d63ffc4a', 'fresh']], ['small', ['array', '<i4', [10], 'eee5b0893685', 'fresh']]], [['ids', ['array', '<i8', [2, 2], '1e1a11cce185', 'fresh']], ['mask', ['array', '<i8', [2, 1], '23b8f6f42560', 'fresh']], ['small', ['array', '<i8', [2, 1], '37089f813939', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 3, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['ids', ['array', '<i8', [6, 7], 'b1151a4651e4', 'fresh']], ['mask', ['array', '|b1', [18], '80e4d63ffc4a', 'fresh']], ['small', ['array', '<i4', [10], 'eee5b0893685', 'fresh']]], [['ids', ['array', '<i8', [2, 2], '1e1a11cce185', 'fresh']], ['mask', ['array', '<i8', [2, 1], '23b8f6f42560', 'fresh']], ['small', ['array', '<i8', [2, 1], '37089f813939', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_d2h': 3, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_response_keys': 1}, 'concat_device_calls': 0, 'launches': 6, 'result': ['ok', [[['ids', ['array', '<i8', [6, 7], 'b1151a4651e4', 'fresh']], ['mask', ['array', '|b1', [18], '80e4d63ffc4a', 'fresh']], ['small', ['array', '<i4', [10], 'eee5b0893685', 'fresh']]], [['ids', ['array', '<i8', [2, 2], '1e1a11cce185', 'fresh']], ['mask', ['array', '<i8', [2, 1], '23b8f6f42560', 'fresh']], ['small', ['array', '<i8', [2, 1], '37089f813939', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'padded_varint_few': {
        'cold': [
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 8, 'result': ['ok', [[['x', ['array', '<i8', [8], 'd1b4082d226e', 'fresh']]], [['x', ['array', '<i8', [2, 1], 'a385649cbb41', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 8, 'result': ['ok', [[['x', ['array', '<i8', [8], 'd1b4082d226e', 'fresh']]], [['x', ['array', '<i8', [2, 1], 'a385649cbb41', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 8, 'result': ['ok', [[['x', ['array', '<i8', [8], 'd1b4082d226e', 'fresh']]], [['x', ['array', '<i8', [2, 1], 'a385649cbb41', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_padded_layout': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 8, 'result': ['ok', [[['x', ['array', '<i8', [8], 'd1b4082d226e', 'fresh']]], [['x', ['array', '<i8', [2, 1], 'a385649cbb41', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'padded_varint_range': {
        'cold': [
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_parse_responses_host': 1, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 10, 'result': ['raise', 'OverflowError'], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_parse_responses_host': 1, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 10, 'result': ['raise', 'OverflowError'], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_parse_responses_host': 1, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 10, 'result': ['raise', 'OverflowError'], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_parse_responses_host': 1, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 10, 'result': ['raise', 'OverflowError'], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'padded_varint_rows': {
        'cold': [
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 16, 'result': ['ok', [[['x', ['array', '<i4', [6], 'bc820beafeab', 'fresh']]], [['x', ['array', '<i8', [2, 1], '7590cbf3642e', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 16, 'result': ['ok', [[['x', ['array', '<i4', [6], 'bc820beafeab', 'fresh']]], [['x', ['array', '<i8', [2, 1], '7590cbf3642e', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 16, 'result': ['ok', [[['x', ['array', '<i4', [6], 'bc820beafeab', 'fresh']]], [['x', ['array', '<i8', [2, 1], '7590cbf3642e', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_decode_padded': 1, 'b200tfs_memcpy_h2d': 1, 'b200tfs_padded_layout': 1, 'b200tfs_padded_results': 1, 'b200tfs_parse_responses_host': 2, 'b200tfs_response_keys': 1, 'b200tfs_unpack_outputs_host': 2}, 'concat_device_calls': 0, 'launches': 16, 'result': ['ok', [[['x', ['array', '<i4', [6], 'bc820beafeab', 'fresh']]], [['x', ['array', '<i8', [2, 1], '7590cbf3642e', 'fresh']]], [['spec', 'default', 1, True, '', 'serving_default'], ['spec', 'default', 1, True, '', 'serving_default']]]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'parse': {
        'cold': [
            {'calls': {'b200tfs_parse_responses_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['d', 'scores'], ['o0', 'o1', 'o2', 'o3', 'o4', 'o5', 'o6', 'o7', 'o8'], ['a', 'ids', 'm', 's']]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_parse_responses_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['d', 'scores'], ['o0', 'o1', 'o2', 'o3', 'o4', 'o5', 'o6', 'o7', 'o8'], ['a', 'ids', 'm', 's']]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_parse_responses_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['d', 'scores'], ['o0', 'o1', 'o2', 'o3', 'o4', 'o5', 'o6', 'o7', 'o8'], ['a', 'ids', 'm', 's']]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_parse_responses_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['ok', [['d', 'scores'], ['o0', 'o1', 'o2', 'o3', 'o4', 'o5', 'o6', 'o7', 'o8'], ['a', 'ids', 'm', 's']]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'tensor_protos': {
        'cold': [
            {'calls': {'b200tfs_parse_tensor_protos_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 5, 'result': ['ok', [['array', '<f4', [3, 4], '7b0b2e8fe8a1', 'fresh'], ['array', '<i4', [5], '73d8e2a2d150', 'fresh'], ['array', '<f8', [2, 2], 'f8f5d84cd1d8', 'fresh']]], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_parse_tensor_protos_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 5, 'result': ['ok', [['array', '<f4', [3, 4], '7b0b2e8fe8a1', 'fresh'], ['array', '<i4', [5], '73d8e2a2d150', 'fresh'], ['array', '<f8', [2, 2], 'f8f5d84cd1d8', 'fresh']]], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_parse_tensor_protos_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 5, 'result': ['ok', [['array', '<f4', [3, 4], '7b0b2e8fe8a1', 'fresh'], ['array', '<i4', [5], '73d8e2a2d150', 'fresh'], ['array', '<f8', [2, 2], 'f8f5d84cd1d8', 'fresh']]], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_parse_tensor_protos_host': 1, 'b200tfs_unpack_outputs_host': 1}, 'concat_device_calls': 0, 'launches': 5, 'result': ['ok', [['array', '<f4', [3, 4], '7b0b2e8fe8a1', 'fresh'], ['array', '<i4', [5], '73d8e2a2d150', 'fresh'], ['array', '<f8', [2, 2], 'f8f5d84cd1d8', 'fresh']]], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
    'tensor_protos_strict': {
        'cold': [
            {'calls': {'b200tfs_parse_tensor_protos_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_parse_tensor_protos_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': False, 'stats': [0, 0, 0]},
        ],
        'warm': [
            {'calls': {'b200tfs_parse_tensor_protos_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [0, 0, 0]},
            {'calls': {'b200tfs_parse_tensor_protos_host': 1}, 'concat_device_calls': 0, 'launches': 1, 'result': ['raise', 'ValueError'], 'seen_varints': True, 'stats': [0, 0, 0]},
        ],
    },
}
