"""The 16-bit float references of the oracle, pinned against numpy / ml_dtypes / the reference before they judge the kernels.

wire_oracle.narrow_f32 is what ``tensor_proto_to_ndarray(...).astype(np.float16 / bfloat16)`` gives (the decoded float32 is
quiet already); wire_oracle.widen_16 is what the reference puts on the wire for a float16 / bfloat16 tensor encoded as
DT_FLOAT; wire_oracle.int_to_half is the reference's reading of DT_HALF half_val integers as values.
"""
import numpy as np
import pytest

import cast_sweep
from oracle import ref_port, wire_oracle


def _astype_bits(bits, np_dtype):
    with np.errstate(over="ignore", invalid="ignore"):
        return bits.view(np.float32).astype(np_dtype).view(np.uint16)


def _check_narrow(bits):
    import ml_dtypes

    nan = cast_sweep.is_nan(bits)
    for np_dtype in (np.float16, ml_dtypes.bfloat16):
        got = wire_oracle.narrow_f32(bits.view(np.float32), np_dtype).view(np.uint16)
        want = _astype_bits(cast_sweep.quiet(bits), np_dtype)
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, (np.dtype(np_dtype).name, [(hex(bits[i]), hex(got[i]), hex(want[i])) for i in bad[:8]])
        if np_dtype is np.float16:   # the documented NaN rule, spelled out
            w = cast_sweep.quiet(bits[nan])
            assert np.array_equal(got[nan], ((w >> 16) & 0x8000) | 0x7E00 | ((w >> 13) & 0x3FF))
        else:
            assert np.array_equal(got[nan], np.where(bits[nan] >> 31 != 0, 0xFFC0, 0x7FC0))


def test_narrow_f32_matches_astype_on_the_sweep():
    bits = np.array(cast_sweep.f32_patterns())
    assert bits.size > 1_000_000
    assert cast_sweep.is_nan(bits).sum() > 1000 and (bits & 0x7F800000 == 0).sum() > 1000
    _check_narrow(bits)


def test_narrow_f32_edges_spelled_out():
    f16 = lambda w: int(wire_oracle.narrow_f32(np.array([w], dtype=np.uint32).view(np.float32), np.float16).view(np.uint16)[0])
    assert f16(0x477FE000) == 0x7BFF and f16(0x477FEFFF) == 0x7BFF and f16(0x477FF000) == 0x7C00   # 65504 / tie -> inf
    assert f16(0x33000000) == 0x0000 and f16(0x33000001) == 0x0001 and f16(0x80000001) == 0x8000  # 2^-25 tie -> +0; -tiny -> -0
    assert f16(0x7FC00001) == 0x7E00 and f16(0xFFC12345) == 0xFE09 and f16(0x7F800001) == 0x7E00


def test_widen_16_matches_astype_on_every_pattern():
    for x in (cast_sweep.all_f16(), cast_sweep.all_bf16()):
        got = wire_oracle.widen_16(x).view(np.uint32)
        assert np.array_equal(got, cast_sweep.quiet(x.astype(np.float32).view(np.uint32))), x.dtype
        nan = np.isnan(x.astype(np.float32))
        assert nan.sum() == (2046 if x.dtype == np.float16 else 254)


def test_int_to_half_matches_the_reference():
    from tensorflow.core.framework import tensor_pb2, tensor_shape_pb2, types_pb2

    v = np.array(cast_sweep.int32_sweep())
    assert v.size > 300_000 and v.min() == -(1 << 31) and v.max() == (1 << 31) - 1
    tp = tensor_pb2.TensorProto(dtype=types_pb2.DT_HALF,
                                tensor_shape=tensor_shape_pb2.TensorShapeProto(dim=[tensor_shape_pb2.TensorShapeProto.Dim(size=v.size)]))
    tp.half_val.extend(v.tolist())
    with np.errstate(over="ignore"):
        want = ref_port.decode_tensor_proto(tp.SerializeToString())
    got = wire_oracle.int_to_half(v)
    assert want.dtype == np.float16
    bad = np.flatnonzero(got.view(np.uint16) != want.view(np.uint16))
    assert bad.size == 0, [(int(v[i]), hex(got.view(np.uint16)[i]), hex(want.view(np.uint16)[i])) for i in bad[:8]]


@cast_sweep.EXHAUSTIVE
def test_narrow_f32_matches_astype_on_every_float32(request):
    import os
    from concurrent.futures import ThreadPoolExecutor

    cast_sweep.require_exhaustive(request.config)
    chunk = 1 << 24

    def one(c):          # numpy's casts and the oracle's ctypes call release the GIL: chunks run in parallel
        _check_narrow(np.arange(c * chunk, (c + 1) * chunk, dtype=np.uint64).astype(np.uint32))

    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as pool:
        for f in [pool.submit(one, c) for c in range((1 << 32) // chunk)]:
            f.result()
