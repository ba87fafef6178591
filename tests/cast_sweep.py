"""Seeded value sets for the 16-bit float conversions (tests/test_casts_cpu.py, tests/test_casts_gpu.py).

``f32_patterns()`` holds about 1.2 M float32 bit patterns chosen where a narrowing to float16 or bfloat16 goes wrong: the
rounding cut of both formats at every exponent (exact, just below, at and just above the half-way point, with an even
and an odd kept LSB), the float16 overflow edge, the bfloat16 overflow band, float16-subnormal results, float32
subnormals, NaNs of every kind, infinities and zeros, and a million random patterns.  The hand-picked specials come
first, so a small rotation moves them through the head of a payload.
"""
import functools
import warnings

import numpy as np
import pytest

SEED = 20261015


def _tie_mantissas(drop, rng):
    """23-bit mantissas around a rounding cut that drops the low `drop` bits (drop <= 23)."""
    kept = 23 - drop
    half = 1 << (drop - 1)
    lows = {0, 1, half - 1, half, half + 1, (1 << drop) - 1}
    highs = {0}
    if kept > 1:
        hb = kept - 1
        highs |= {(1 << hb) - 1, 1 << (hb - 1), int("10" * hb, 2) & ((1 << hb) - 1), int("01" * hb, 2) & ((1 << hb) - 1)}
        highs |= {int(v) for v in rng.integers(0, 1 << hb, 2)}
    out = []
    for h in sorted(highs):
        for lsb in ((0, 1) if kept else (0,)):
            for lo in sorted(lows):
                out.append((((h << 1) | lsb) << drop | lo) & 0x7FFFFF)
    return out


@functools.lru_cache(maxsize=None)
def f32_patterns() -> np.ndarray:
    """uint32 bit patterns (read-only)."""
    rng = np.random.default_rng(SEED)
    parts = []
    # NaNs: signalling and quiet, both signs, payload 1 / top bit only / all ones, and random payloads
    nan_m = [1, 0x200000, 0x3FFFFF, 0x1FFF, 0x2000, 0x400000, 0x400001, 0x600000, 0x7FFFFF, 0x401FFF, 0x402000]
    nan_m += [int(v) for v in rng.integers(1, 1 << 23, 500)]
    for s in (0, 0x80000000):
        parts.append(np.array([s | 0x7F800000 | m for m in nan_m], dtype=np.uint64))
    # infinities, zeros, float32 subnormals, extremes of both 16-bit formats
    edge = [0x7F800000, 0x00000000, 0x00000001, 0x00000002, 0x007FFFFF, 0x00400000, 0x00008000, 0x00010000, 0x00018000,
            0x7F7FFFFF, 0x7F7F8000, 0x7F7F7FFF, 0x477FE000, 0x477FEFFF, 0x477FF000, 0x477FF001, 0x47800000, 0x38800000,
            0x387FC000, 0x33800000, 0x33000000, 0x33000001, 0x32FFFFFF, 0x00800000, 0x3F800000]
    edge += [int(v) for v in rng.integers(1, 1 << 23, 200)]                          # random float32 subnormals
    for s in (0, 0x80000000):
        parts.append(np.array([s | w for w in edge], dtype=np.uint64))
    # every exponent x the rounding cut of float16 (13 dropped bits) and bfloat16 (16); float16-subnormal results
    # (float32 exponents 102..112 drop 14..24 bits of the significand, the hidden bit included)
    cuts = []
    for e in range(256):
        drops = {13, 16}
        if 102 <= e <= 113:
            drops.add(13 + 113 - e)
        for drop in sorted(drops):
            if drop <= 23:
                ms = _tie_mantissas(drop, rng)
            else:                                                            # the hidden bit is the half-way bit
                ms = [0, 1, 0x7FFFFF, 0x400000] + [int(v) for v in rng.integers(0, 1 << 23, 4)]
            cuts += [(e << 23) | m for m in ms]
    cuts = np.array(cuts, dtype=np.uint64)
    parts += [cuts, cuts | 0x80000000]
    # every float32 from 65504 (largest float16) to 65536; the bfloat16 overflow band
    f16_edge = np.arange(0x477FE000, 0x47800001, dtype=np.uint64)
    bf16_band = np.arange(0x7F7F0000, 0x7F800000, dtype=np.uint64)
    parts += [f16_edge, f16_edge | 0x80000000, bf16_band, bf16_band | 0x80000000]
    parts.append(rng.integers(0, 1 << 32, 1 << 20, dtype=np.uint64))
    out = np.concatenate(parts).astype(np.uint32)
    out.flags.writeable = False
    return out


def is_nan(bits: np.ndarray) -> np.ndarray:
    return (bits & 0x7FFFFFFF) > 0x7F800000


def quiet(bits: np.ndarray) -> np.ndarray:
    """float32 NaNs made quiet (sign and payload kept), as a trip through a C double leaves them."""
    bits = np.asarray(bits, dtype=np.uint32)
    return np.where(is_nan(bits), bits | np.uint32(0x400000), bits).astype(np.uint32)


def all_f16() -> np.ndarray:
    return np.arange(1 << 16, dtype=np.uint32).astype(np.uint16).view(np.float16)


def all_bf16() -> np.ndarray:
    import ml_dtypes

    return np.arange(1 << 16, dtype=np.uint32).astype(np.uint16).view(ml_dtypes.bfloat16)


@functools.lru_cache(maxsize=None)
def int32_sweep() -> np.ndarray:
    """int32 half_val values for the DT_HALF quirk: all of [-70000, 70000] (float16's whole finite range and its overflow),
    2^k + {-2..2}, and every float16 spacing point 2^k + j * 2^(k-11) (the odd j are ties) +- 1, both signs, and the int32 ends."""
    vals = [np.arange(-70000, 70001, dtype=np.int64)]
    k = np.arange(0, 32, dtype=np.int64)
    p = np.int64(1) << k
    vals += [p + d for d in range(-2, 3)]
    for kk in range(12, 32):
        grid = (np.int64(1) << kk) + np.arange(2048, dtype=np.int64) * (np.int64(1) << (kk - 11))
        vals += [grid - 1, grid, grid + 1]
    v = np.concatenate(vals)
    v = np.concatenate([v, -v, [-(1 << 31), (1 << 31) - 1]])
    v = v[(v >= -(1 << 31)) & (v < (1 << 31))]
    out = np.unique(v).astype(np.int32)
    out.flags.writeable = False
    return out


# The tests over all 2^32 float32 patterns carry this mark and take minutes: `-m exhaustive` selects them, and
# require_exhaustive() skips them in every other run.  The suite's settings do not register the mark, hence no warning here.
with warnings.catch_warnings():
    warnings.simplefilter("ignore", pytest.PytestUnknownMarkWarning)
    EXHAUSTIVE = pytest.mark.exhaustive


def require_exhaustive(config) -> None:
    if "exhaustive" not in (config.option.markexpr or ""):
        pytest.skip("every float32 pattern: select with -m exhaustive")


def rotated(x: np.ndarray, case: int, step: int = 3) -> np.ndarray:
    """x rotated by `step * case` elements, so successive cases put other values into a payload's head and tail."""
    return np.roll(x, step * case)
