"""Pins tests/move_ref.py - the byte references and the geometry model of the fixed-width move engine - against whole messages
from the CPU oracle and the protobuf runtime, and checks the model's invariants exhaustively: the tiles of every payload
partition its bytes, and no vector load leaves the 16-byte blocks of the source (a load there cannot fault)."""
import os
import re

import ml_dtypes
import numpy as np
import pytest

import cast_sweep
import move_ref as M
from oracle import wire_oracle
from tensorflow.core.framework import tensor_pb2

CSRC = M._CSRC


def f32_classes():
    """sNaN and qNaN of both signs and several payloads, +-inf, denormals, +-0, normals."""
    w = [0x7F800001, 0x7FBFFFFF, 0x7FC00000, 0x7FC00001, 0x7FFFFFFF, 0xFF800001, 0xFFBFFFFF, 0xFFC00000, 0xFFFFFFFF,
         0x7F800000, 0xFF800000, 0x00000001, 0x007FFFFF, 0x80000001, 0x807FFFFF, 0x00000000, 0x80000000, 0x3F800000, 0xC0490FDB]
    return np.array(w, dtype=np.uint32)


def payload(wire, raw):
    """The one place `raw` lies in `wire`."""
    at = wire.find(raw)
    assert at >= 0 and wire.find(raw, at + 1) < 0
    return wire[at: at + len(raw)]


def test_constants_match_the_sources():
    with open(os.path.join(CSRC, "kernels.cu")) as f:
        cu = f.read()
    assert re.search(r"constexpr uint32_t kStageVecs = kStageVecsHost;", cu)
    assert re.search(r"constexpr uint32_t kU = 4, kRun = 32 \* kU", cu)           # body_narrow_q's round
    assert re.search(r"constexpr uint32_t kU = 8;", cu)                              # body_widen's round
    assert (M.K_SMALL_MAX, M.K_MOVE_THREADS, M.K_STAGE_VECS, M.K_STAGE_BUFS) == (2048, 256, 2048, 2)
    assert M.ROUND_ALIGNED == M.ROUND_SHIFT == 2048 and M.ROUND_NARROW == 1024
    assert M.K_INLINE_PLAN_BYTES < 4096


def test_plan_struct_sizes_match_plan_h():
    """The plan image model counts bytes of the structs as plan.h lays them out: fields and their order are pinned here."""
    with open(os.path.join(CSRC, "plan.h")) as f:
        h = re.sub(r"//[^\n]*", "", f.read())
    def fields(name):
        body = re.search(r"struct %s \{(.*?)\};" % name, h, re.S).group(1)
        return re.findall(r"(const uint8_t\*|uint8_t\*|const uint32_t\*|uint64_t|uint32_t)\s+([\w\[\], ]+);", body)
    size = {"const uint8_t*": 8, "uint8_t*": 8, "const uint32_t*": 8, "uint64_t": 8, "uint32_t": 4}
    def nbytes(name):
        total = 0
        for t, names in fields(name):
            for nm in names.split(","):
                m = re.search(r"\[(\d+)\]", nm)
                total += size[t] * (int(m.group(1)) if m else 1)
        return total
    assert (nbytes("PlanHeader"), nbytes("MoveItem"), nbytes("TileRef"), nbytes("SmallItem")) == \
        (M.PLAN_HEADER_BYTES, M.MOVE_ITEM_BYTES, M.TILE_REF_BYTES, M.SMALL_ITEM_BYTES)
    assert M.plan_image(1, 0, 0, 0) == 112 and M.inline_plan(M.plan_image(2, 8, 6, 400))
    assert not M.inline_plan(M.plan_image(95, 0, 0, 0))


def test_quiet_matches_the_oracle_on_every_float32_class():
    bits = np.concatenate([f32_classes(), cast_sweep.f32_patterns()[:4096]])
    x = bits.view(np.float32)
    want = M.out_bytes(M.QUIET_SRC, x.tobytes())
    # encode: the oracle quiets sNaN on the wire unless asked to keep it
    wire = wire_oracle.encode_tensor_proto(x)
    assert payload(wire, want) == want
    assert np.array_equal(np.frombuffer(want, np.uint32), cast_sweep.quiet(bits))
    assert wire_oracle.encode_tensor_proto(x, keep_snan=True).find(M.out_bytes(M.COPY, x.tobytes())) > 0
    # decode: the oracle's float32 values are the quieted ones
    resp = wire_oracle.build_predict_response([("x", x)], keep_snan=True)
    assert wire_oracle.decode_predict_response(resp)["x"].tobytes() == M.out_bytes(M.QUIET_DST, x.tobytes())
    # exactly the NaNs change, and only by the quiet bit
    w = np.frombuffer(want, np.uint32)
    nan = (bits & 0x7FFFFFFF) > 0x7F800000
    assert np.array_equal(w[~nan], bits[~nan]) and np.all(w[nan] == bits[nan] | 0x400000)


def test_bool_bytes_0_to_255_match_the_oracle_and_the_protobuf_runtime():
    raw = np.arange(256, dtype=np.uint8)
    want = M.out_bytes(M.BOOL, raw.tobytes())
    assert want == bytes([0] + [1] * 255)
    tp = tensor_pb2.TensorProto(dtype=10)
    tp.tensor_shape.dim.add(size=256)
    tp.bool_val.extend([bool(b) for b in raw])
    assert wire_oracle.encode_tensor_proto(raw.view(np.bool_)) == tp.SerializeToString()
    assert payload(tp.SerializeToString(), want) == want


def test_narrow_and_widen_reuse_the_oracle():
    bits = np.concatenate([f32_classes(), cast_sweep.f32_patterns()[:20000]])
    for op, dt in ((M.F2H, np.float16), (M.F2B, ml_dtypes.bfloat16)):
        got = np.frombuffer(M.out_bytes(op, bits.tobytes()), np.uint16)
        assert np.array_equal(got, wire_oracle.narrow_f32(bits.view(np.float32), dt).view(np.uint16))
        # NaNs come out quiet with the sign kept
        nan = (bits & 0x7FFFFFFF) > 0x7F800000
        assert np.all((got[nan] & 0x7FFF) >= (0x7E00 if dt is np.float16 else 0x7FC0)) and np.array_equal(got[nan] >> 15, bits[nan] >> 31)
    for op, x in ((M.H2F, cast_sweep.all_f16()), (M.B2F, cast_sweep.all_bf16())):
        got = M.out_bytes(op, x.tobytes())
        assert got == wire_oracle.widen_16(x).tobytes()
        wire = wire_oracle.encode_tensor_proto(x, wire_dtype=np.float32)
        assert payload(wire, got) == got


def test_gather_reads_a_row_of_unpacked_elements():
    x = np.arange(37, dtype=np.uint32).view(np.float32)
    row = b"".join(b"\x2d" + x[i: i + 1].tobytes() for i in range(x.size))
    assert M.gather(row[1:], 4, 5, 4 * x.size).tobytes() == x.tobytes()


def test_pick_vec_per_tile():
    assert M.pick_vec_per_tile(132, 4 << 20, 32768) == 2048
    assert M.pick_vec_per_tile(132, 1 << 30, 65536) == 4096
    assert M.pick_vec_per_tile(132, 64 << 20, 65536) == 4096
    assert M.pick_vec_per_tile(132, 40 << 20, 65536) == 4096 and M.pick_vec_per_tile(132, 30 << 20, 65536) == 2048
    assert M.pick_vec_per_tile(132, 1, 65536, override=32800) == 2050
    assert M.pick_vec_per_tile(132, 1, 32768, override=32) == 2 and M.pick_vec_per_tile(132, 1, 32768, override=95) == 4
    assert M.pick_vec_per_tile(132, 0, 32768, override=1) == 2


def check_geometry(g, vpt):
    """Every invariant of one payload's geometry."""
    n = g.n_out
    if g.fast:
        assert g.head + 16 * g.nvec + g.tail == n and g.tail >= 0 and g.nvec >= 0
        if g.kind == "widen":
            assert g.nvec % 2 == 0 and g.head == 0
    # the writes of the tiles partition [0, n_out), head only in tile 0, tail only in the last tile
    w = g.writes(vpt)
    covered = 0
    nt = M.tiles_for(n, vpt)
    for t, a, b in sorted(w, key=lambda r: r[1]):
        assert a == covered and b > a, (g.__dict__, w)
        covered = b
    assert covered == n
    if g.fast:
        tiles = g.tiles(vpt)
        assert sum(x[2] for x in tiles) == g.nvec and len(tiles) == nt
        v = 0
        for t, v0, cnt, _ in tiles:
            assert cnt == 0 or v0 == v
            v += cnt
        if g.tail:
            assert any(t == nt - 1 and b == n for t, a, b in w)
        if g.kind == "widen":
            assert all(x[2] % 2 == 0 for x in tiles)
    # loads stay inside the source's 16-byte blocks
    lo, hi = g.read_window()
    for a, b in g.loads(vpt):
        assert lo <= a and b <= hi and (a & 15) == 0 and (b & 15) == 0, (g.__dict__, a, b)
    st = g.staged(vpt) if g.dec else None
    if st:
        for t, chunks in st:
            for c, nc, nbytes, off, parity in chunks:
                a = g.src_body - g.k + off
                assert lo <= a and a + nbytes <= hi and nbytes % 16 == 0, (g.__dict__, c, nc)


def lengths(vpt, tiles=3):
    """[0, tiles * vpt * 16 + 64] at small vpt; the edges of tiles, rounds and staged chunks at the real ones."""
    T = 16 * vpt
    if vpt <= 16:
        return range(0, tiles * T + 65)
    edges = {0, 1, 15, 16, 17, M.K_SMALL_MAX - 1, M.K_SMALL_MAX, M.K_SMALL_MAX + 1}
    for m in range(1, tiles + 1):
        edges |= {m * T + d for d in range(-17, 18)} | {m * T + d for d in (-32, -48, 32, 48, 64)}
    for r in (M.ROUND_ALIGNED, M.ROUND_NARROW, M.K_STAGE_VECS):
        for m in range(1, vpt // r + 1):
            edges |= {16 * m * r + d for d in (-16, -1, 0, 1, 16, 32)}
    return sorted(e for e in edges if e >= 0)


@pytest.mark.parametrize("vpt", [2, 4, 6, 2048, 2050, 4096, 6144, 10240, 16384])
def test_geometry_invariants_at_every_phase(vpt):
    base_s, base_d = 1 << 20, 1 << 24
    ns = lengths(vpt)
    hits = set()
    for op, dec, esz in ((M.COPY, True, 1), (M.QUIET_DST, False, 4), (M.BOOL, False, 1), (M.QUIET_SRC, False, 4),
                         (M.H2F, False, 2), (M.F2H, False, 4)):
        for k in range(16):
            for dph in range(16):
                for n in ns:
                    if (op == M.H2F and (n % 4 or k % 2)) or (op == M.F2H and n % 2):
                        continue
                    g = M.Geometry(base_s + k, base_d + dph, n, op, dec=dec)
                    check_geometry(g, vpt)
                    hits.add((op, g.body()))
                    if dec and g.fast:
                        st = g.staged(vpt)
                        assert st is not None and all(len(ch) <= -(-vpt // M.K_STAGE_VECS) for _, ch in st)
    assert (M.COPY, "aligned") in hits and all((M.COPY, "shifted%d" % q) in hits for q in range(4))
    assert (M.H2F, "widen") in hits and (M.F2H, "narrow") in hits and (M.F2H, "narrow3") in hits


def test_staged_chunks_of_the_documented_tile_sizes():
    """B200TFS_TILE_BYTES 32800 / 65536 / 98304 / 163840 / 262144: 2 chunks with a 2-vector second one, 2, 3, 5, 8 chunks;
    chunk 2 and later of a three-or-more chunk tile refill a buffer and wait on parity 1."""
    want = {32800: (2, 2), 65536: (2, 2048), 98304: (3, 2048), 163840: (5, 2048), 262144: (8, 2048)}
    for tb, (chunks, last) in want.items():
        vpt = M.pick_vec_per_tile(132, 1 << 30, 65536, override=tb)
        g = M.Geometry(1 << 20, 1 << 24, 16 * vpt * 2 + 5, M.COPY, dec=True)
        ch = g.staged(vpt)[0][1]
        assert len(ch) == chunks and ch[-1][1] == last, tb
        assert any(p == 1 for *_, p in ch) == (chunks > 2), tb
