"""A seeded, deterministic corpus of malformed and same-length-mutated PredictResponse / TensorProto records, and the
expected results of each, for the differential decode tests (tests/test_decode_mutants_cpu.py, tests/test_decode_mutants_gpu.py).

Every seed is a valid record.  Its mutants are:
  - every truncation (large seeds: every one near a framing byte and a seeded sample of the rest), made by shortening
    rec_len over the UNCHANGED buffer, so the bytes past the end are the record's real continuation bytes;
  - every single-bit flip of every framing byte (framing: every byte outside the value runs the host walker locates);
  - bit flips inside the value runs: all of them for small records, a seeded sample for large ones (every one:
    value_flips(), behind the suite's `exhaustive` mark);
  - every length prefix set to +-1 and +-128 of its value, and re-encoded one byte longer (non-minimal);
  - the continuation bit of the last byte of each packed-varint run set, and that of the byte before it cleared;
  - same-length framing edits that parse to another table: a key byte, a dim within its varint length, float <-> double,
    a model_spec byte, a chunk boundary moved.  These must miss the framing template of the seed.

The expected table of a record is what the tag walker (min-tfs-client_b200/csrc/walker.h) computes for it on the host
(tests/native); tests/test_decode_mutants_cpu.py pins that reference against the protobuf runtime and the reference's
algorithm (oracle/ref_port.py) on the whole corpus.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from dataclasses import dataclass, field
from typing import Iterator, List, Optional

import numpy as np

import golden_util as G
from cast_sweep import EXHAUSTIVE, require_exhaustive  # noqa: F401 - the opt-in mark of the suite's long sweeps
from min_tfs_client import _native as N

HERE = os.path.dirname(os.path.abspath(__file__))


# ---- the host build of the walker --------------------------------------------------------------------------------------
class SpillEntry(C.Structure):
    _fields_ = [("kind", C.c_uint32), ("seq", C.c_uint32), ("run", N.Run)]


SPILL_DIM, SPILL_RUN = 1, 2
_walker = None


def walker():
    global _walker
    if _walker is None:
        subprocess.run(["make", "-s", "-C", os.path.join(HERE, "native")], check=True)
        L = C.CDLL(os.path.join(HERE, "native", "_build", "libwalker_host.so"))
        L.wh_parse_response.restype = C.c_int
        L.wh_parse_response.argtypes = [C.c_void_p, C.c_uint64, C.c_int, C.POINTER(N.Output), C.POINTER(C.c_int), C.POINTER(N.ModelSpec),
                                        C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)]
        L.wh_parse_tensor.restype = C.c_int
        L.wh_parse_tensor.argtypes = [C.c_void_p, C.c_uint64, C.POINTER(N.Output), C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)]
        assert L.wh_sizeof_output() == C.sizeof(N.Output) and L.wh_sizeof_spill_entry() == C.sizeof(SpillEntry)
        _walker = L
    return _walker


@dataclass
class Walk:
    """What the walker tabulates for one record: status, outputs (complete dims and value runs), spec."""
    status: int
    outs: List[N.Output]
    spec: N.ModelSpec
    dims: List[List[int]]
    runs: List[List[tuple]]     # (off, len, count, stride, field)


def _full(o, spill):
    """Every dim and every value run of one output: inline ones first, then its spill entries in order."""
    dims = [int(o.dims[k]) for k in range(min(o.rank, N.MAX_RANK))]
    runs = [(int(r.off), int(r.len), int(r.count), int(r.stride), int(r.field)) for r in (o.runs[k] for k in range(o.n_inline))]
    for e in spill:
        if e.seq != o.spill_seq:
            continue
        if e.kind == SPILL_DIM and len(dims) < o.rank:
            dims.append(int(e.run.off))
        elif e.kind == SPILL_RUN and e.run.field == o.value_field and len(runs) < o.n_runs:
            runs.append((int(e.run.off), int(e.run.len), int(e.run.count), int(e.run.stride), int(e.run.field)))
    return dims, runs


def walk(buf: bytes, rec_len: int, tensor=False, max_outputs=16, spill=True) -> Walk:
    """The host walker over buf[:rec_len] (buf is passed whole: a walk that reads past rec_len sees real bytes).  With
    `spill`, runs again with a spill area as large as the record wants, as the two-phase parse does; without it, a record
    that wants one reports B200TFS_E_SPILL, as the single-launch decode's walk does."""
    L = walker()
    raw = C.create_string_buffer(bytes(buf), max(len(buf), 1))
    cap = 0
    for _ in range(2):
        area = (SpillEntry * max(cap, 1))()
        used = C.c_uint32()
        spec = N.ModelSpec()
        if tensor:
            outs = (N.Output * 1)()
            st = L.wh_parse_tensor(raw, rec_len, outs, area if cap else None, cap, C.byref(used))
            cnt = 1 if st == N.OK else 0
        else:
            outs = (N.Output * (max_outputs + 1))()
            n = C.c_int()
            st = L.wh_parse_response(raw, rec_len, max_outputs, outs, C.byref(n), C.byref(spec), area if cap else None, cap, C.byref(used))
            cnt = n.value
        if st != N.E_SPILL or not spill:
            break
        cap = used.value
    entries = list(area[: min(used.value, cap)]) if cap else []
    keep = [N.Output.from_buffer_copy(outs[k]) for k in range(cnt)]
    full = [_full(o, entries) for o in keep]
    return Walk(st, keep, spec, [f[0] for f in full], [f[1] for f in full])


def spec_text(rec: bytes, s: N.ModelSpec):
    """The model_spec a table points at, as values: name, signature, label and version."""
    return (rec[s.name_off: s.name_off + s.name_len], rec[s.signature_off: s.signature_off + s.signature_len],
            rec[s.label_off: s.label_off + s.label_len], int(s.has_version), int(s.version))


# ---- value bytes --------------------------------------------------------------------------------------------------------
FIXED = {1: np.float32, 2: np.float64}       # the fixed-width dtypes of the corpus (8 / 18, complex, never appear)
VARINT_DTYPES = {3, 4, 5, 6, 9, 10, 17, 22, 23}


def run_bytes(buf: bytes, runs) -> bytes:
    return b"".join(buf[off + q * stride: off + q * stride + ln] for off, ln, count, stride, _ in runs for q in range(count))


def quiet_f32(raw: bytes) -> bytes:
    u = np.frombuffer(raw, dtype=np.uint32).copy()
    u[(u & 0x7FFFFFFF) > 0x7F800000] |= 0x00400000
    return u.tobytes()


def fixed_values(buf: bytes, w: Walk, k: int) -> bytes:
    """The bytes a decode writes for fixed-width output k: its value runs in wire order, float32 NaNs quieted."""
    raw = run_bytes(buf, w.runs[k])
    return quiet_f32(raw) if w.outs[k].dtype == 1 else raw


def malformed_varints(buf: bytes, w: Walk, k: int) -> bool:
    """The varint decode kernels' structural check, restated: every varint of every run ends within ten bytes."""
    if not (w.outs[k].flags & N.OF_VARINT):
        return False
    for off, ln, count, stride, _ in w.runs[k]:
        for q in range(count):
            run = 0
            for b in buf[off + q * stride: off + q * stride + ln]:
                run = run + 1 if b & 0x80 else 0
                if run >= 10:
                    return True
            if run:
                return True
    return False


def value_ranges(w: Walk):
    """[start, end) byte ranges the walker locates as values: the runs of every output and tensor_content."""
    out = []
    for o, runs in zip(w.outs, w.runs):
        for off, ln, count, stride, _ in runs:
            out += [(off + q * stride, off + q * stride + ln) for q in range(count)]
        if o.content_len:
            out.append((int(o.content_off), int(o.content_off + o.content_len)))
    return out


# ---- the framing template, restated (tpl.h tpl_learn and the verdict of decode_fused_body) -------------------------------
@dataclass
class Template:
    rec_len: int
    chunks: List[tuple]        # (wire_off, len, is_varint), by wire offset
    framing: bytes


def template_of(buf: bytes, max_framing=256, max_chunks=4) -> Optional[Template]:
    """The template the single-launch decode learns from this (clean) record, or None when it does not qualify."""
    w = walk(buf, len(buf), max_outputs=N.FUSED_MAX_OUTPUTS, spill=False)
    if w.status != N.OK:
        return None
    ch = []
    for o, runs in zip(w.outs, w.runs):
        if o.status not in (N.OK, N.E_SHAPE, N.E_KEY) or o.flags & (N.OF_UNPACKED | N.OF_SPILLED):
            return None
        for off, ln, count, _, _ in runs:
            if count != 1:
                return None
            ch.append((off, ln, bool(o.flags & N.OF_VARINT)))
        if o.content_len:
            ch.append((int(o.content_off), int(o.content_len), False))
    ch.sort()
    if len(ch) > max_chunks:
        return None
    value = set()
    for off, ln, _ in ch:
        value.update(range(off, off + ln))
    framing = bytes(b for i, b in enumerate(buf) if i not in value)
    if len(framing) > max_framing:
        return None
    return Template(len(buf), ch, framing)


def verdict(t: Template, buf: bytes, rec_len: int) -> bool:
    """Does the record carry the template's framing: same length, the same bytes outside the template's value chunks, and
    every packed-varint chunk still ending on a terminator?"""
    if rec_len != t.rec_len:
        return False
    value = np.zeros(rec_len, dtype=bool)
    for off, ln, _ in t.chunks:
        value[off: off + ln] = True
    rec = np.frombuffer(bytes(buf[:rec_len]), dtype=np.uint8)
    if rec[~value].tobytes() != t.framing:
        return False
    return all(not (ln and rec[off + ln - 1] & 0x80) for off, ln, v in t.chunks if v)


def layout(outs: List[N.Output], stride: int, cast: int = 0) -> List[N.Output]:
    """tpl.h tpl_layout_outputs restated: every fixed-width output that decoded cleanly gets a 256-byte aligned range of
    the record's slot, in table order; with a narrowing cast DT_FLOAT outputs take two bytes per element."""
    got, cursor = [], 0
    for o in outs:
        o = N.Output.from_buffer_copy(o)
        if o.status == N.OK and o.n_elems and o.dtype in FIXED:
            if cast and o.dtype == 1:
                o.dst_bytes = o.n_elems * 2
            cursor = (cursor + 255) & ~255
            if cursor + o.dst_bytes > stride:
                o.status = N.E_SIZE
            else:
                o.dst_off = cursor
                cursor += o.dst_bytes
        got.append(o)
    return got


# ---- seeds --------------------------------------------------------------------------------------------------------------
ld, vi, entry, tproto, mspec, shape = G.ld, G.vi, G.entry, G.tproto, G.mspec, G.shape


def f32(n, seed):
    return np.random.default_rng(seed).standard_normal(n).astype(np.float32)


def f64(n, seed):
    return np.random.default_rng(seed).standard_normal(n)


def packed_varints(vals):
    return b"".join(vi(int(v)) for v in vals)


def out(key, dtype, dims, body):
    return entry(key, tproto(dtype, dims, body))


@dataclass
class Seed:
    name: str
    wire: bytes
    tensor: bool = False
    edits: List[tuple] = field(default_factory=list)    # (label, bytes of the same length)


def _key_edit(wire, key):
    """The same record with the last byte of its first occurrence of `key` changed (another valid key)."""
    at = wire.index(key.encode()) + len(key) - 1
    b = bytearray(wire)
    b[at] = ord("Z") if b[at] != ord("Z") else ord("Y")
    return bytes(b)


def _spec_edit(wire, name=b"default"):
    at = wire.rindex(name) + len(name) - 1
    b = bytearray(wire)
    b[at] ^= 1
    return bytes(b)


def _sized_key(target_len, build):
    """A key length that makes build(key) exactly target_len bytes long."""
    for k in range(1, 400):
        if len(build("q" * k)) == target_len:
            return "q" * k
    raise ValueError(target_len)


def seeds() -> List[Seed]:
    S = []
    x7, x8 = f32(7, 1), f32(8, 2)
    x8[3] = np.array([0x7F800001], dtype=np.uint32).view(np.float32)[0]     # a signalling NaN: the decode quiets it
    w = out("scores", 1, [7], ld(0x2A, x7.tobytes())) + mspec()
    S.append(Seed("f32", w, edits=[("key", _key_edit(w, "scores")), ("dim", out("scores", 1, [6], ld(0x2A, x7.tobytes())) + mspec()),
                                   ("spec", _spec_edit(w))]))
    w = mspec() + out("y", 1, [2, 4], ld(0x2A, x8.tobytes()))
    S.append(Seed("f32_spec_first", w, edits=[
        ("key", mspec() + out("z", 1, [2, 4], ld(0x2A, x8.tobytes()))),
        ("dims", mspec() + out("y", 1, [4, 2], ld(0x2A, x8.tobytes()))),
        ("dtype", mspec() + out("y", 2, [1, 4], ld(0x32, x8.tobytes()))),
        ("spec", _spec_edit(w))]))
    d = f64(15, 3)
    w = out("d", 2, [3, 5], ld(0x32, d.tobytes())) + mspec()
    S.append(Seed("f64", w, edits=[("dims", out("d", 2, [5, 3], ld(0x32, d.tobytes())) + mspec()),
                                   ("dtype", out("d", 1, [6, 5], ld(0x2A, d.tobytes())) + mspec()), ("key", _key_edit(w, "d"))]))
    # several outputs: float, int64 and bool varints, a string output, unknown fields (inside a TensorProto and at the top level), a group
    ids = np.array([0, 1, 127, 128, 300, -5], dtype=np.int64)
    strs = ld(0x42, b"ab") + ld(0x42, b"xyz")
    unknown = b"\xB8\x06\x07" + b"\xC1\x06" + b"\x01" * 8 + b"\xAA\x06\x03abc"
    group = b"\xC3\x06\xB8\x06\x01\xC4\x06"

    def multi(a_dims=(4,), ids_key="ids", m_dims=(5,)):
        return (out("a", 1, list(a_dims), ld(0x2A, x7[:4].tobytes()) + b"\xF8\x01\x05")
                + unknown + out(ids_key, 9, [6], ld(0x52, packed_varints(ids.view(np.uint64))))
                + out("m", 10, list(m_dims), ld(0x5A, bytes([1, 0, 1, 1, 0]))) + group
                + entry("s", tproto(7, [2], strs)) + mspec())
    w = multi()
    S.append(Seed("multi", w, edits=[("key", multi(ids_key="idt")), ("dim", multi(m_dims=(4,))), ("dims", multi(a_dims=(3,))),
                                     ("spec", _spec_edit(w))]))
    # float_val in two packed occurrences; the edit moves the boundary between them (same bytes, same total length)
    x12 = f32(12, 4).tobytes()
    w = out("v", 1, [12], ld(0x2A, x12[:16]) + ld(0x2A, x12[16:]))
    S.append(Seed("split", w, edits=[("boundary", out("v", 1, [12], ld(0x2A, x12[:20]) + ld(0x2A, x12[20:]))),
                                     ("boundary2", out("v", 1, [12], ld(0x2A, x12[:4]) + ld(0x2A, x12[4:])))]))
    # a float output that also carries packed int_val: the table drops those runs, yet the runtime refuses the message when
    # one of their varints is malformed (the walk used to accept such a record; found by this corpus on big_f32, whose
    # float_val tag 0x2A flipped to 0x3A turns 80 KB of floats into a malformed int_val).  Here: 2^63 takes ten bytes, and
    # flipping the top bit of its last one makes a varint longer than ten bytes, while the run still ends on a terminator
    w = out("fv", 1, [4], ld(0x3A, packed_varints([1, 300, 2 ** 63, 5])) + ld(0x2A, x8[:4].tobytes())) + mspec()
    S.append(Seed("foreign_varint", w, edits=[("key", out("fw", 1, [4], ld(0x3A, packed_varints([1, 300, 2 ** 63, 5])) + ld(0x2A, x8[:4].tobytes()))
                                                + mspec())]))
    # more than 16 dims and more than 8 value runs: both spill (the two-phase parse re-runs with a spill area)
    x45 = f32(45, 5).tobytes()
    body, at = b"", 0
    for k in range(1, 10):
        body += ld(0x2A, x45[at * 4: (at + k) * 4])
        at += k
    S.append(Seed("spill", out("deep", 1, [1] * 16 + [45], body) + mspec()))
    # longer than 256 B with framing bytes in three and more 128-byte lines: the device walk evicts cache lines
    ka, kb, kc = "first_" + "a" * 30, "second_" + "b" * 24, "third_" + "c" * 20
    a40, b20, c40 = f32(40, 6), f64(20, 7), f32(40, 8)

    def evict(kc=kc, b_dims=(4, 5), name=b"model_" + b"n" * 40):
        return (out(ka, 1, [40], ld(0x2A, a40.tobytes())) + out(kb, 2, list(b_dims), ld(0x32, b20.tobytes()))
                + out(kc, 1, [40], ld(0x2A, c40.tobytes())) + mspec(name=name))
    w = evict()
    S.append(Seed("evict", w, edits=[("key", evict(kc=kc[:-1] + "d")), ("dims", evict(b_dims=(5, 4))),
                                     ("spec", evict(name=b"model_" + b"n" * 39 + b"m"))]))
    # records of 127..129 and 255..257 bytes: the last byte on either side of a line boundary (offsets cover every phase)
    for target in (127, 128, 129, 255, 256, 257):
        def build(k, target=target):
            return out(k, 1, [9], ld(0x2A, f32(9, target).tobytes())) + mspec()
        k = _sized_key(target, build)
        S.append(Seed(f"len{target}", build(k), edits=[("key", _key_edit(build(k), k))]))
    # tensor_content (opaque to the walk, never moved by the single-launch decode) next to a typed float output
    c8 = f32(8, 9).tobytes()
    S.append(Seed("content", out("c", 1, [2, 4], ld(0x22, c8)) + out("f", 1, [2], ld(0x2A, x7[:2].tobytes())) + mspec()))
    # large: two and more 32 KB tiles
    big = f32(20000, 10)
    w = out("image", 1, [100, 200], ld(0x2A, big.tobytes())) + mspec()
    S.append(Seed("big_f32", w, edits=[("dims", out("image", 1, [200, 100], ld(0x2A, big.tobytes())) + mspec()),
                                       ("key", _key_edit(w, "image")), ("spec", _spec_edit(w))]))
    bd = f64(10000, 11)
    w = out("dd", 2, [100, 100], ld(0x32, bd.tobytes())) + mspec()
    S.append(Seed("big_f64", w, edits=[("dtype", out("dd", 1, [100, 100], ld(0x2A, bd.tobytes())) + mspec()), ("key", _key_edit(w, "dd"))]))
    bi = G.make_array({"gen": "varint_mix", "seed": 12, "dtype": "int64", "shape": [12000]})
    w = out("tokens", 9, [12000], ld(0x52, packed_varints(bi.view(np.uint64)))) + mspec()
    S.append(Seed("big_i64", w, edits=[("key", _key_edit(w, "tokens"))]))
    # bare TensorProtos
    S.append(Seed("t_f32", tproto(1, [3, 4], ld(0x2A, f32(12, 13).tobytes())), tensor=True))
    S.append(Seed("t_f64_content", tproto(2, [2, 2], ld(0x22, f64(4, 14).tobytes())), tensor=True))
    S.append(Seed("t_i32", tproto(3, [5], ld(0x3A, packed_varints(np.array([1, -1, 300, 0, 2 ** 31 - 1], np.int64).view(np.uint64))))
                  + b"\xF8\x01\x05", tensor=True))
    S.append(Seed("t_big_f32", tproto(1, [9000], ld(0x2A, f32(9000, 15).tobytes())), tensor=True))
    for s in S:
        for label, e in s.edits:
            assert len(e) == len(s.wire) and e != s.wire, (s.name, label)
    return S


# ---- length prefixes (a plain scan of the schema the seeds use) ---------------------------------------------------------
_SUB = {"resp": {1: "entry", 2: "spec"}, "entry": {2: "tensor"}, "tensor": {2: "shape"}, "shape": {2: "dim"}, "spec": {2: "i64"},
        "dim": {}, "i64": {}}


def _rv(b, p):
    v = s = 0
    while True:
        x = b[p]
        p += 1
        v |= (x & 0x7F) << s
        s += 7
        if not x & 0x80:
            return v, p


def length_prefixes(wire: bytes, kind: str):
    """(offset, byte count, value) of every length prefix in a valid record."""
    found = []

    def scan(lo, hi, msg):
        p = lo
        depth = 0
        while p < hi:
            tag, p = _rv(wire, p)
            wt = tag & 7
            if wt == 0:
                _, p = _rv(wire, p)
            elif wt == 1:
                p += 8
            elif wt == 5:
                p += 4
            elif wt == 3:
                depth += 1
            elif wt == 4:
                depth -= 1
            elif wt == 2:
                q = p
                n, p = _rv(wire, p)
                found.append((q, p - q, n))
                if depth == 0 and (tag >> 3) in _SUB[msg]:
                    scan(p, p + n, _SUB[msg][tag >> 3])
                p += n

    scan(0, len(wire), kind)
    return found


# ---- mutants ------------------------------------------------------------------------------------------------------------
@dataclass
class Mutant:
    seed: str
    kind: str
    buf: bytes       # the bytes the record lies in (a truncation keeps the seed's bytes past rec_len)
    rec_len: int
    tensor: bool = False

    @property
    def record(self) -> bytes:
        return self.buf[: self.rec_len]


SMALL = 2048      # records up to this long get every truncation and every value-bit flip


def mutants(s: Seed) -> List[Mutant]:
    w = s.wire
    n = len(w)
    rng = np.random.default_rng(sum(w[:64]) + n)
    base = walk(w, n, tensor=s.tensor)
    assert base.status == N.OK, s.name
    value = np.zeros(n, dtype=bool)
    for a, b in value_ranges(base):
        value[a:b] = True
    framing = np.flatnonzero(~value)
    vbytes = np.flatnonzero(value)
    got: List[Mutant] = []

    def add(kind, buf, rec_len=None):
        got.append(Mutant(s.name, kind, bytes(buf), len(buf) if rec_len is None else rec_len, s.tensor))

    # truncations over the unchanged buffer
    if n <= SMALL:
        cuts = range(n)
    else:
        near = set()
        for f in framing:
            near.update(range(max(int(f) - 2, 0), min(int(f) + 3, n)))
        cuts = sorted(near | set(int(c) for c in rng.integers(0, n, 48)))
    for c in cuts:
        add("truncate", w, c)
    # single-bit flips of every framing byte
    for i in framing:
        for bit in range(8):
            b = bytearray(w)
            b[i] ^= 1 << bit
            add("framing_flip", b)
    # value-bit flips (every one of a large seed: value_flips(), which yields them as it goes)
    if vbytes.size:
        if n <= SMALL:
            picks = [(int(i), bit) for i in vbytes for bit in range(8)]
        else:
            picks = [(int(vbytes[j]), int(bit)) for j, bit in zip(rng.integers(0, vbytes.size, 96), rng.integers(0, 8, 96))]
            picks += [(int(vbytes[0]), 7), (int(vbytes[-1]), 7), (int(vbytes[-1]), 0)]
        for i, bit in picks:
            b = bytearray(w)
            b[i] ^= 1 << bit
            add("value_flip", b)
    # length prefixes: +-1, +-128, one byte longer than minimal
    for at, nb, v in length_prefixes(w, "tensor" if s.tensor else "resp"):
        for dv in (-128, -1, 1, 128):
            if v + dv >= 0:
                add("length", w[:at] + vi(v + dv) + w[at + nb:])
        long = bytearray(vi(v))
        long[-1] |= 0x80
        add("length_nonminimal", w[:at] + bytes(long) + b"\x00" + w[at + nb:])
    # the terminator of each packed-varint run
    for o, runs in zip(base.outs, base.runs):
        if not o.flags & N.OF_VARINT:
            continue
        for off, ln, count, stride, _ in runs:
            if count == 1 and ln:
                b = bytearray(w)
                b[off + ln - 1] |= 0x80
                add("varint_end_set", b)
                if ln > 1 and w[off + ln - 2] & 0x80:
                    b = bytearray(w)
                    b[off + ln - 2] &= 0x7F
                    add("varint_end_clear", b)
    for label, e in s.edits:
        add("same_len_" + label, e)
    seen, uniq = set(), []
    for m in got:
        k = (m.buf, m.rec_len)
        if k in seen or (m.rec_len == n and m.buf == w):
            continue
        seen.add(k)
        uniq.append(m)
    return uniq


def value_flips(s: Seed) -> Iterator[Mutant]:
    """Every single-bit flip of every value byte of a seed, one at a time (a large seed has some 640 000 of them)."""
    base = walk(s.wire, len(s.wire), tensor=s.tensor)
    for a, b in value_ranges(base):
        for i in range(a, b):
            for bit in range(8):
                buf = bytearray(s.wire)
                buf[i] ^= 1 << bit
                yield Mutant(s.name, "value_flip", bytes(buf), len(buf), s.tensor)


def corpus():
    """[(seed, [mutants])] for every seed."""
    return [(s, mutants(s)) for s in seeds()]
