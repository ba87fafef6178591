"""Every kernel route that converts between float32 and float16 / bfloat16, bit for bit against the oracle's references.

The values are the sweep of tests/cast_sweep.py: rounding ties of both formats at every exponent, the overflow edges,
subnormal results and inputs, NaNs of every kind, infinities, zeros and random patterns; for the widening and the 16-bit
fields, all 65 536 patterns of each format.  Key lengths 0-15 move the float32 payload through every byte phase of the
wire and the sweep is rotated per case, so the specials pass through the ragged heads and tails as well as the vector
bodies.  Narrowed outputs must equal ``wire_oracle.narrow_f32`` (numpy / ml_dtypes ``astype`` of the reference's decoded
float32, NaNs quiet), widened inputs ``wire_oracle.widen_16``, DT_HALF values read strictly ``wire_oracle.int_to_half``.
"""
import ctypes as C

import ml_dtypes
import numpy as np
import pytest

import cast_sweep
from devutil import Dev, tensor_struct
from min_tfs_client import _native as N
from oracle import ref_port, wire_oracle
from test_device_api_gpu import _decode_cast
from test_host_pipeline_gpu import _decode_host, _encode_host, _pipelined

pytestmark = pytest.mark.gpu

NP16 = {19: np.float16, 14: ml_dtypes.bfloat16}
CASTS = [19, 14, 1]      # fp16, bf16, and the cast off (float32 out: the same data pins sNaN quieting)
HEAD = 1 << 19           # every hand-picked pattern of the sweep and some random ones: 2 MiB of float32


def _sweep(case, n=None):
    bits = cast_sweep.f32_patterns()
    return cast_sweep.rotated(bits[:n] if n else bits, case).view(np.float32)


def _want(x, cast):
    """Expected output bytes of a float32 payload x decoded with cast (1: no cast)."""
    if cast == 1:
        return cast_sweep.quiet(x.view(np.uint32)).view(np.float32)
    return wire_oracle.narrow_f32(x, NP16[cast])


def _same(got, want, src, what):
    """got / want: output element arrays (16- or 32-bit); src: the float32 inputs, for the message."""
    g, w = np.frombuffer(bytes(got), dtype=want.dtype).view(np.uint16 if want.itemsize == 2 else np.uint32), want.view(
        np.uint16 if want.itemsize == 2 else np.uint32)
    assert g.size == w.size, (what, g.size, w.size)
    bad = np.flatnonzero(g != w)
    assert bad.size == 0, (what, bad.size, [(int(i), hex(src.view(np.uint32)[i]), hex(g[i]), hex(w[i])) for i in bad[:6]])


def _same_wire(got, want, what):
    """Byte strings equal; on a difference, report where instead of diffing megabytes."""
    if got != want:
        g, w = np.frombuffer(got, np.uint8), np.frombuffer(want, np.uint8)
        n = min(g.size, w.size)
        first = ([int(i) for i in np.flatnonzero(g[:n] != w[:n])[:1]] or [n])[0]
        pytest.fail(f"{what}: {len(got)} vs {len(want)} bytes, first difference at {first}: "
                    f"{got[first: first + 8].hex()} vs {want[first: first + 8].hex()}")


def _stats(dev):
    a, b, c = C.c_uint64(), C.c_uint64(), C.c_uint64()
    N.check(dev.lib.b200tfs_decode_stats(dev.ctx, C.byref(a), C.byref(b), C.byref(c)))
    return a.value + b.value, c.value          # (served by a template, walked)


def _launches(dev):
    v = C.c_uint64()
    N.check(dev.lib.b200tfs_kernel_launches(dev.ctx, C.byref(v)))
    return v.value


def _out_bytes(slot, o):
    return slot[o.dst_off: o.dst_off + o.dst_bytes]


# ---- narrowing: the single-launch decode ---------------------------------------------------------------------------------
@pytest.mark.parametrize("cast", CASTS)
def test_fused_decode_walk_and_template(cast):
    """R1: a fresh context walks the record; R2: the same record again takes the framing template.  Key lengths 0-15."""
    for key_len in range(16):
        x = _sweep(key_len, HEAD)
        key = "k" * key_len
        wire = wire_oracle.build_predict_response([(key, x)], keep_snan=True)
        want = _want(x, cast)
        dev = Dev(0)
        try:
            for rep in range(2):
                t0, w0 = _stats(dev)
                slot, outs, n_outs, status = _decode_cast(dev, [wire], (x.nbytes + 511) & ~255, cast)
                t1, w1 = _stats(dev)
                assert status[0] == 0 and n_outs[0] == 1 and outs[0].n_elems == x.size
                assert (w1 - w0, t1 - t0) == ((1, 0) if rep == 0 else (0, 1)), (key_len, rep)
                _same(_out_bytes(slot[0], outs[0]), want, x, (cast, key_len, rep))
        finally:
            dev.close()


@pytest.mark.parametrize("cast", CASTS)
def test_host_wire_pipelined_decode(cast):
    """R3: a host-resident wire of several MiB (b200tfs_decode_responses_host_async), misaligned host pointer too.  Uncast,
    the sliced, pipelined path cuts the payload at places unrelated to the patterns; a narrowing call stays one launch over
    the template the host walked."""
    dev = Dev(0)
    try:
        N.check(dev.lib.b200tfs_set_decode_cast(dev.ctx, cast))
        for case, (key_len, shift) in enumerate([(0, 0), (3, 0), (6, 5), (13, 2)]):
            x = _sweep(case)
            wire = wire_oracle.build_predict_response([("y" * key_len, x)], keep_snan=True)
            assert len(wire) >= 1 << 20
            p0 = _pipelined(dev)
            out, outs, n_outs, status, keep = _decode_host(dev, wire, (x.nbytes + 2303) & ~255, shift)
            assert status == 0 and n_outs == 1 and _pipelined(dev) == p0 + (cast == 1)
            _same(_out_bytes(out, outs[0]), _want(x, cast), x, (cast, key_len, shift))
    finally:
        dev.close()


@pytest.mark.parametrize("cast", CASTS)
def test_staged_batch_decode(cast):
    """R4: 96 responses x 602 KB of float32 (the geometry of the staged batch kernels), cut from the tiled sweep."""
    P = 150528
    big = np.resize(cast_sweep.f32_patterns(), 96 * P).view(np.float32).reshape(96, P)
    want = _want(big.reshape(-1), cast).reshape(96, P)
    batch = [wire_oracle.build_predict_response([("image", big[i])], keep_snan=True) for i in range(96)]
    dev = Dev(0)
    try:
        for rep in range(2):
            slot, outs, n_outs, status = _decode_cast(dev, batch, (P * want.itemsize + 255) & ~255, cast)
            assert all(status[i] == 0 and n_outs[i] == 1 for i in range(96))
            for i in range(96):
                _same(_out_bytes(slot[i], outs[i * N.FUSED_MAX_OUTPUTS]), want[i], big[i], (cast, rep, i))
    finally:
        dev.close()


@pytest.mark.parametrize("cast", CASTS)
def test_three_launch_batch_decode(cast):
    """R5: a narrowing batch of equal-length records (> 4 MiB) whose length the context knows: verify launch, guarded move,
    fallback.  In the last pass record 5 has the same length but another key, so the fallback launch walks it.  Uncast,
    the same batches go through the single-launch decode."""
    both = np.concatenate([cast_sweep.f32_patterns(), cast_sweep.rotated(cast_sweep.f32_patterns(), 1)])
    n = 16
    per = both.size // n
    recs = both[: n * per].view(np.float32).reshape(n, per)
    want = _want(recs.reshape(-1), cast).reshape(n, per)
    def wire(i, key="image"):
        return wire_oracle.build_predict_response([(key, recs[i])], keep_snan=True)
    batch = [wire(i) for i in range(n)]
    assert sum(len(w) for w in batch) >= 4 << 20
    dev = Dev(0)
    try:
        l0 = _launches(dev)
        for rep in range(3):
            if rep == 2:
                batch[5] = wire(5, key="imagf")
            slot, outs, n_outs, status = _decode_cast(dev, batch, (per * want.itemsize + 255) & ~255, cast)
            for i in range(n):
                assert status[i] == 0 and n_outs[i] == 1, (rep, i)
                _same(_out_bytes(slot[i], outs[i * N.FUSED_MAX_OUTPUTS]), want[i], recs[i], (cast, rep, i))
        if cast != 1:
            assert _launches(dev) - l0 >= 1 + 3 + 3, "the second and third pass run as three launches each"
    finally:
        dev.close()


# ---- narrowing: two-phase parse + unpack ---------------------------------------------------------------------------------
def _parse_unpack(dev, wire, cast, dst_shift):
    """b200tfs_parse_responses + b200tfs_unpack_outputs into a device pointer dst_shift bytes past a 256-byte boundary."""
    arena = dev.upload(np.frombuffer(wire, dtype=np.uint8))
    off, ln = (C.c_uint64 * 1)(0), (C.c_uint64 * 1)(len(wire))
    outs = (N.Output * 4)()
    n_outs, specs, status = (C.c_int32 * 1)(), (N.ModelSpec * 1)(), (C.c_int32 * 1)()
    N.check(dev.lib.b200tfs_parse_responses(dev.ctx, arena, 1, off, ln, 4, outs, n_outs, specs, status))
    assert status[0] == 0 and n_outs[0] == 1
    o = outs[0]
    nbytes = int(o.n_elems) * (4 if cast == 1 else 2)
    base = dev.malloc(nbytes + 512)
    N.check(dev.lib.b200tfs_memset(dev.ctx, base, 0xEE, nbytes + 512))
    dst = (C.c_void_p * 1)(base + dst_shift)
    st = (C.c_int32 * 1)()
    N.check(dev.lib.b200tfs_unpack_outputs(dev.ctx, arena, 1, outs, None, dst, (C.c_int32 * 1)(cast), st))
    assert st[0] == 0
    got = dev.download(base, nbytes + 512)
    assert (got[:dst_shift] == 0xEE).all() and (got[dst_shift + nbytes:] == 0xEE).all()     # nothing written outside
    for p in dev.allocs[-2:]:
        dev.lib.b200tfs_free(dev.ctx, p)
    del dev.allocs[-2:]
    return o, got[dst_shift: dst_shift + nbytes]


@pytest.mark.parametrize("cast", CASTS)
def test_two_phase_unpack_at_every_destination_phase(cast):
    """R6: destination pointers offset by 0-15 bytes (odd offsets take the byte generator for the whole payload), with the
    key length moving the source phase at the same time."""
    dev = Dev(0)
    try:
        for shift in range(16):
            x = _sweep(shift, HEAD)
            wire = wire_oracle.build_predict_response([("s" * ((shift * 7) % 16), x)], keep_snan=True)
            o, got = _parse_unpack(dev, wire, cast, shift)
            _same(got, _want(x, cast), x, (cast, shift))
    finally:
        dev.close()


def _unpacked_float_val_response(x, key):
    """A response whose float_val is written element by element (tag + 4 bytes each): a gathered source row."""
    def uv(v):
        out = bytearray()
        while v >= 0x80:
            out.append((v & 0x7F) | 0x80)
            v >>= 7
        out.append(v)
        return bytes(out)
    dim = b"\x08" + uv(x.size)
    shape = b"\x12" + uv(len(dim)) + dim
    vals = (np.frombuffer(b"\x2d", np.uint8).repeat(x.size).reshape(-1, 1))
    body = np.concatenate([vals, x.view(np.uint8).reshape(-1, 4)], axis=1).tobytes()
    tp = b"\x08\x01\x12" + uv(len(shape)) + shape + body
    entry = b"\x0a" + uv(len(key)) + key + b"\x12" + uv(len(tp)) + tp
    return b"\x0a" + uv(len(entry)) + entry


@pytest.mark.parametrize("cast", CASTS)
def test_unpacked_float_val_row(cast):
    """R7: unpacked float_val elements (one 5-byte field each): the unpack reads them through a gathered source view."""
    dev = Dev(0)
    try:
        for case, shift in enumerate((0, 1, 6)):
            x = _sweep(case, 1 << 17)
            wire = _unpacked_float_val_response(x, b"row")
            assert list(wire_oracle.decode_predict_response(wire)) == ["row"]
            o, got = _parse_unpack(dev, wire, cast, shift)
            assert o.n_runs >= 1 and o.runs[0].stride == 5 and o.runs[0].len == 4
            _same(got, _want(x, cast), x, (cast, shift))
    finally:
        dev.close()


def test_python_out_dtypes(codec):
    """R8: decode_predict_response(out_dtypes=...) covering every float output (single launch) and only some of them
    (two-phase fallback); both against the oracle."""
    f, g = _sweep(1, HEAD), _sweep(2)[-99991:]
    ids = np.arange(50, dtype=np.int64)
    resp = wire_oracle.build_predict_response([("f", f), ("g", g), ("ids", ids)], keep_snan=True)
    for cast, np_dt in NP16.items():
        every = codec.decode_predict_response(resp, out_dtypes={"f": np_dt, "g": np_dt})[0]
        part = codec.decode_predict_response(resp, out_dtypes={"f": np_dt})[0]
        for got, name, src in ((every["f"], "f", f), (every["g"], "g", g), (part["f"], "f part", f)):
            assert got.dtype == np.dtype(np_dt)
            _same(got.tobytes(), wire_oracle.narrow_f32(src, np_dt), src, (cast, name))
        _same(part["g"].tobytes(), _want(g, 1), g, (cast, "g uncast"))
        assert every["ids"].tobytes() == ids.tobytes()


# ---- widening: float16 / bfloat16 sources encoded as DT_FLOAT -------------------------------------------------------------
def _all16(np_dt, reps, case):
    x = cast_sweep.all_f16() if np_dt is np.float16 else cast_sweep.all_bf16()
    return cast_sweep.rotated(np.tile(x, reps), case)


@pytest.mark.parametrize("np_dt", [np.float16, ml_dtypes.bfloat16], ids=["f16", "bf16"])
def test_widen_host_numpy(codec, np_dt):
    """W1: host numpy input to encode_predict_requests(wire_dtype="DT_FLOAT"), key lengths moving the payload's phase."""
    for key_len in range(8):
        x = _all16(np_dt, 2, key_len)
        key = "x" * key_len
        wire = codec.encode_predict_request("default", {key: x}, 1, wire_dtype="DT_FLOAT")
        want = wire_oracle.encode_predict_request("default", 1, [(key, x)], wire_dtype=np.float32)
        assert wire_oracle.widen_16(x).tobytes() in want
        _same_wire(wire, want, key_len)


def _encode_on_device(dev, inputs, deferred=False):
    """One request; inputs: [(key, array, src byte offset, wire dtype)] uploaded at `offset` past a 256-byte boundary."""
    keep, ts = [], []
    for k, a, shift, wire_dt in inputs:
        raw = np.zeros(a.nbytes + 16, dtype=np.uint8)
        raw[shift: shift + a.nbytes] = a.reshape(-1).view(np.uint8)
        p = dev.upload(raw)
        t, dims = tensor_struct(p + shift, a, key=k.encode(), wire_dtype=wire_dt)
        keep.append((t, dims))
        ts.append(t)
    arr = (N.Tensor * len(ts))(*ts)
    req = N.Request(model_name=b"default", model_name_len=7, has_version=1, order=N.ORDER_UPB, version=1, n_inputs=len(ts),
                    flags=0, inputs=arr)
    rq = (N.Request * 1)(req)
    need = C.c_uint64()
    if not deferred:
        N.check(dev.lib.b200tfs_measure(dev.ctx, len(ts), arr))
    N.check(dev.lib.b200tfs_request_arena_size(1, rq, C.byref(need)))
    arena = dev.malloc(need.value)
    off, ln = (C.c_uint64 * 1)(), (C.c_uint64 * 1)()
    if deferred:
        N.check(dev.lib.b200tfs_encode_requests_async(dev.ctx, 1, rq, arena, need.value))
        N.check(dev.lib.b200tfs_encode_results(dev.ctx, 1, off, ln))
    else:
        N.check(dev.lib.b200tfs_encode_requests(dev.ctx, 1, rq, arena, need.value, off, ln))
    dev.sync()
    return dev.download(arena, need.value)[off[0]: off[0] + ln[0]].tobytes()


@pytest.mark.parametrize("np_dt", [np.float16, ml_dtypes.bfloat16], ids=["f16", "bf16"])
def test_widen_misaligned_device_sources(np_dt):
    """W2: source pointers at +2 .. +14 bytes through the C ABI, and a second widened input of odd length in the same request,
    whose destination is not 16-byte aligned: both take the byte generator."""
    dev = Dev(0)
    try:
        for case, shift in enumerate(range(2, 16, 2)):
            x = _all16(np_dt, 1, case)
            y = _all16(np_dt, 1, case + 7)[:65536 - 3]
            inputs = [("a", x, shift, 1), ("bb" + "c" * case, y, 16 - shift, 1)]
            got = _encode_on_device(dev, inputs)
            want = wire_oracle.encode_predict_request("default", 1, [(k, a) for k, a, _, _ in inputs], wire_dtype=np.float32)
            _same_wire(got, want, shift)
    finally:
        dev.close()


@pytest.mark.parametrize("np_dt", [np.float16, ml_dtypes.bfloat16], ids=["f16", "bf16"])
def test_widen_torch_device_tensors(codec, np_dt):
    """W3: device-resident torch tensors, through __cuda_array_interface__ (float16 only: it has no bfloat16 type string)
    and through DLPack."""
    torch = pytest.importorskip("torch")

    class DLPackOnly:
        def __init__(self, t):
            self.t = t

        def __dlpack__(self, **kw):
            return self.t.__dlpack__(**kw)

        def __dlpack_device__(self):
            return self.t.__dlpack_device__()

    class CAIOnly:
        def __init__(self, t):
            self.__cuda_array_interface__ = t.__cuda_array_interface__

    x = _all16(np_dt, 2, 5)
    tdt = torch.float16 if np_dt is np.float16 else torch.bfloat16
    t = torch.from_numpy(x.view(np.int16).copy()).cuda().view(tdt)
    torch.cuda.synchronize()
    want = wire_oracle.encode_predict_request("default", 1, [("x", x)], wire_dtype=np.float32)
    views = [DLPackOnly(t)] + ([CAIOnly(t)] if np_dt is np.float16 else [])
    for v in views:
        _same_wire(codec.encode_predict_request("default", {"x": v}, 1, wire_dtype="DT_FLOAT"), want, type(v).__name__)


@pytest.mark.parametrize("np_dt", [np.float16, ml_dtypes.bfloat16], ids=["f16", "bf16"])
def test_widen_pipelined_host_buffers(np_dt):
    """W4: the host-buffer entry point with several MiB of source: the pipelined slices cut through the patterns."""
    dev = Dev(0)
    try:
        for case in range(3):
            x = _all16(np_dt, 16, case)
            p0 = _pipelined(dev)
            got = _encode_host(dev, [("default", 1, [("x" * case, x)])], wire_dtypes={(0, 0): 1})[0]
            assert _pipelined(dev) == p0 + 1
            _same_wire(got, wire_oracle.encode_predict_request("default", 1, [("x" * case, x)], wire_dtype=np.float32), case)
    finally:
        dev.close()


@pytest.mark.parametrize("np_dt", [np.float16, ml_dtypes.bfloat16], ids=["f16", "bf16"])
def test_widen_in_the_deferred_encode(np_dt):
    """W5: b200tfs_encode_requests_async with a packed-varint input in the same request."""
    dev = Dev(0)
    try:
        x = _all16(np_dt, 1, 11)
        ids = (np.arange(5000, dtype=np.int64) * 7919) % 300007 - 150
        got = _encode_on_device(dev, [("x", x, 6, 1), ("ids", ids, 0, 9)], deferred=True)
        want = wire_oracle.encode_predict_request("default", 1, [("x", x.astype(np.float32)), ("ids", ids)])
        _same_wire(got, want, "deferred")
    finally:
        dev.close()


# ---- 16-bit fields: half_val varints ----------------------------------------------------------------------------------
@pytest.mark.parametrize("np_dt", [np.float16, ml_dtypes.bfloat16], ids=["f16", "bf16"])
def test_half_val_bit_patterns_round_trip(codec, np_dt):
    """H1: every float16 / bfloat16 pattern as half_val varints: the encode equals the oracle, the tolerant decode gives
    back the same bits."""
    x = _all16(np_dt, 1, 3)
    wire = codec.encode_predict_request("default", {"h": x}, 1)
    _same_wire(wire, wire_oracle.encode_predict_request("default", 1, [("h", x)]), "encode")
    resp = wire_oracle.build_predict_response([("h", x)])
    back = codec.decode_predict_response(resp)[0]["h"]
    assert back.dtype == np.dtype(np_dt)
    _same_wire(back.view(np.uint16).tobytes(), x.view(np.uint16).tobytes(), "decode")


def test_half_val_values_strict():
    """H2: the int32 sweep as DT_HALF half_val read with strict=True (the reference's quirk: the integers are VALUES):
    decode_tensor_protos and decode_predict_response against ref_port and int_to_half."""
    from min_tfs_client.codec import Codec
    from tensorflow.core.framework import tensor_pb2, tensor_shape_pb2, types_pb2
    from tensorflow_serving.apis import predict_pb2

    v = np.array(cast_sweep.int32_sweep())
    tp = tensor_pb2.TensorProto(dtype=types_pb2.DT_HALF,
                                tensor_shape=tensor_shape_pb2.TensorShapeProto(dim=[tensor_shape_pb2.TensorShapeProto.Dim(size=v.size)]))
    tp.half_val.extend(v.tolist())
    tp_wire = tp.SerializeToString()
    resp = predict_pb2.PredictResponse()
    resp.outputs["h"].CopyFrom(tp)
    resp_wire = resp.SerializeToString()
    with np.errstate(over="ignore"):
        ref = ref_port.decode_tensor_proto(tp_wire)
    want = wire_oracle.int_to_half(v)
    assert ref.view(np.uint16).tobytes() == want.view(np.uint16).tobytes()
    codec = Codec(0)
    try:
        for got in (codec.decode_tensor_protos([tp_wire], strict=True)[0], codec.decode_predict_response(resp_wire, strict=True)[0]["h"]):
            assert got.dtype == np.float16 and got.shape == v.shape
            bad = np.flatnonzero(got.view(np.uint16) != want.view(np.uint16))
            assert bad.size == 0, [(int(v[i]), hex(got.view(np.uint16)[i]), hex(want.view(np.uint16)[i])) for i in bad[:6]]
    finally:
        codec.close()


# ---- every float32 -----------------------------------------------------------------------------------------------------
@cast_sweep.EXHAUSTIVE
@pytest.mark.parametrize("cast", [19, 14])
def test_fused_decode_every_float32(request, cast):
    """All 2^32 float32 patterns through the single-launch decode on a fresh context (the walk), 256 MiB per response.
    The next response and its expected output are built on the host while the GPU decodes the current one."""
    from concurrent.futures import ThreadPoolExecutor

    cast_sweep.require_exhaustive(request.config)
    chunk = 1 << 26

    def prepare(c):
        x = np.arange(c * chunk, (c + 1) * chunk, dtype=np.uint64).astype(np.uint32).view(np.float32)
        return x, wire_oracle.build_predict_response([("y", x)], keep_snan=True), wire_oracle.narrow_f32(x, NP16[cast])

    with ThreadPoolExecutor(max_workers=1) as pool:
        nxt = pool.submit(prepare, 0)
        for c in range((1 << 32) // chunk):
            x, wire, want = nxt.result()
            if c + 1 < (1 << 32) // chunk:
                nxt = pool.submit(prepare, c + 1)
            dev = Dev(0)
            try:
                slot, outs, n_outs, status = _decode_cast(dev, [wire], x.size * 2 + 256, cast)
                assert status[0] == 0 and n_outs[0] == 1
                _same(_out_bytes(slot[0], outs[0]), want, x, (cast, c))
            finally:
                dev.close()
