"""Classify, Regress and MultiInference responses built to put chosen fields on the edges of the warp entry finder
(csrc/example_resp_kernels.cuh, xr_warp_entries), and a restatement of the finder's schedule that says which edges a case
reaches.  Test infrastructure, like example_ref.py: the decode tests hold the kernels against FromString on these cases, and the
restatement shows that the cases reach what they are named for.

The finder walks a message body [lo, hi) of a record at device address `rec`:
  - a window starts at s (s0 = lo) and covers L = min(256, hi - s) byte positions;
  - the chain runs from s: each member's end is where the next one starts; it stops at the first member that ends at or past
    s + L, is malformed, or is a group (the exit);
  - the next window starts at the exit's end, or at the end of the group, which lane 0 skips with the serial walk (nesting
    deeper than 16 is malformed);
  - the body is staged 4 KB at a time from gb = (rec + s) & ~15, restaged when rec + min(hi, s + 288) > gb + 4096.
Pointer doubling marks at most 128 chain members in a window; every member but the exit takes at least two bytes, so a window
never holds more.
"""
import struct
from dataclasses import dataclass, field
from typing import List, Optional, Tuple

import numpy as np

import example_response_corpus as X
import multi_inference_corpus as M
from example_response_corpus import CLASSIFY, EGROUP, I32, I64, LEN, RAW, REGRESS, SGROUP, VARINT, f32, serialize, varint

WIN, STAGE, MARGIN, GROUP_DEPTH = 256, 4096, 32, 16
ERR, GROUP = "err", "group"


# ---- the restatement ---------------------------------------------------------------------------------------------------------
def _varint_at(b: bytes, p: int, hi: int, most: int = 10):
    """(value, end) of the varint at p, or None when it runs past hi or over `most` bytes (bits past 64 fall off)"""
    v = 0
    for i in range(most):
        if p + i >= hi:
            return None
        x = b[p + i]
        v |= (x & 0x7F) << (7 * i)
        if not x & 0x80:
            return v & (2 ** 64 - 1), p + i + 1
    return None


def _tag_at(b, p, hi):
    r = _varint_at(b, p, hi, 5)
    if r is None or r[0] > 0xFFFFFFFF or r[0] >> 3 == 0:
        return None
    return r


def _after_tag(b: bytes, tag: int, q: int, hi: int):
    """(end, entry body or None) of a non-group field whose tag ends at q; end is ERR or GROUP"""
    wt = tag & 7
    if wt == I64:
        return (q + 8, None) if hi - q >= 8 else (ERR, None)
    if wt == I32:
        return (q + 4, None) if hi - q >= 4 else (ERR, None)
    if wt == SGROUP:
        return GROUP, None
    if wt not in (VARINT, LEN):
        return ERR, None
    v = _varint_at(b, q, hi)
    if v is None:
        return ERR, None
    n, q = v
    if wt == VARINT:
        return q, None
    if n > 0x7FFFFFFF or n > hi - q:
        return ERR, None
    return q + n, ((q, n) if tag == (1 << 3 | LEN) else None)


def field_end(b: bytes, p: int, hi: int):
    """(end, entry body (off, len) or None) of the field at p of a body ending at hi; end is ERR or GROUP (xr_field_end)"""
    t = _tag_at(b, p, hi)
    return (ERR, None) if t is None else _after_tag(b, t[0], t[1], hi)


def skip_group(b: bytes, p: int, hi: int):
    """end of the group whose start tag is at p (walker.h skip_field), or ERR"""
    t = _tag_at(b, p, hi)
    if t is None:
        return ERR
    open_ = [t[0] >> 3]
    p = t[1]
    while open_:
        if p >= hi:
            return ERR
        t = _tag_at(b, p, hi)
        if t is None:
            return ERR
        tag, p = t
        wt = tag & 7
        if wt == SGROUP:
            if len(open_) >= GROUP_DEPTH:
                return ERR
            open_.append(tag >> 3)
        elif wt == EGROUP:
            if open_[-1] != tag >> 3:
                return ERR
            open_.pop()
        else:
            e, _ = _after_tag(b, tag, p, hi)
            if e in (ERR, GROUP):
                return ERR
            p = e
    return p


@dataclass
class Member:
    start: int           # record offset
    end: object          # record offset, ERR or GROUP
    s: int               # the window it lies in
    win: int             # that window's index
    k: int               # window-relative position (start - s)


@dataclass
class Schedule:
    entries: List[Tuple[int, int]] = field(default_factory=list)   # (off, len) of every entry, in wire order
    err: bool = False
    windows: List[Tuple[int, int, int]] = field(default_factory=list)   # (s, L, chain members)
    members: List[Member] = field(default_factory=list)
    stages: List[Tuple[int, int, int]] = field(default_factory=list)    # (s, gb, need) of every staging
    checks: List[Tuple[int, int, int]] = field(default_factory=list)    # (s, gb, need) of every window
    groups: List[Tuple[int, int]] = field(default_factory=list)         # (start, end) of every group lane 0 skipped


def warp_entries(b: bytes, lo: int, hi: int, rec: int = 0) -> Schedule:
    """xr_warp_entries over the body [lo, hi) of the record b at device address rec"""
    S = Schedule()
    s, gb = lo, None
    while s < hi:
        L = min(WIN, hi - s)
        need = min(hi, s + WIN + MARGIN)
        if gb is None or rec + need > gb + STAGE:
            gb = (rec + s) & ~15
            S.stages.append((s, gb, need))
        S.checks.append((s, gb, need))
        k, n = 0, 0
        while True:
            e, body = field_end(b, s + k, hi)
            S.members.append(Member(s + k, e, s, len(S.windows), k))
            n += 1
            if e == ERR:
                S.windows.append((s, L, n))
                S.err = True
                return S
            if e == GROUP:
                g = skip_group(b, s + k, hi)
                S.windows.append((s, L, n))
                if g == ERR:
                    S.err = True
                    return S
                S.groups.append((s + k, g))
                S.members[-1].end = g
                s = g
                break
            if body is not None:
                S.entries.append(body)
            if e - s >= L:
                S.windows.append((s, L, n))
                s = e
                break
            k = e - s
    return S


def _skip_any(b, p, hi):
    e, _ = field_end(b, p, hi)
    return skip_group(b, p, hi) if e == GROUP else e


def results(b: bytes, field_no: int = 1):
    """[(lo, hi)] of every field `field_no` (LEN) at the top level of b, or None when the top level is malformed (xr_next_result)"""
    out, p = [], 0
    while p < len(b):
        t = _tag_at(b, p, len(b))
        if t is None:
            return None
        if t[0] == (field_no << 3 | LEN):
            v = _varint_at(b, t[1], len(b))
            if v is None or v[0] > len(b) - v[1]:
                return None
            out.append((v[1], v[1] + v[0]))
            p = v[1] + v[0]
            continue
        e = _skip_any(b, p, len(b))
        if e == ERR:
            return None
        p = e
    return out


def response_schedules(b: bytes, rec: int = 0):
    """the schedule of every result body of a Classify / Regress response, or None when its top level is malformed"""
    r = results(b)
    return None if r is None else [warp_entries(b, lo, hi, rec) for lo, hi in r]


# ---- the edges a case reaches ------------------------------------------------------------------------------------------------
def edges(case, rec: Optional[int] = None) -> set:
    """Which edges the case reaches, by the restatement: ("start", kind, k) / ("end", kind, e - s) of its target fields,
    ("chain", n[, "odd"]) for windows of 126 to 128 members, ("chain", 128, "ends_at_L"), ("stage", "need_eq" / "need_eq+1"),
    ("restage_rec16", r), ("restage_rec128", r), ("tail", width), ("group_skip", ">4K" / ">8K"), ("err", kind, where),
    ("result2_later_stage",), ("classes", C, "restaged")."""
    rec = case.rec if rec is None else rec
    out = set()
    sch = response_schedules(case.wire, rec) if case.kind in (REGRESS, CLASSIFY) else case.schedules(rec)
    if sch is None:
        return out
    for S in sch:
        by_start = {m.start: m for m in S.members}
        for kind, at in case.targets:
            m = by_start.get(at)
            if m is None:
                continue
            if m.k in (253, 254, 255):
                out.add(("start", kind, m.k))
            if m.k == 0 and m.win > 0 and S.windows[m.win - 1][0] + WIN == m.s:
                out.add(("start", kind, 256))
            if isinstance(m.end, int) and m.end - m.s in (255, 256, 257):
                out.add(("end", kind, m.end - m.s))
            if m.end == ERR:
                if m.win == 0:
                    out.add(("err", kind, "window0"))
                if m.k == 255:
                    out.add(("err", kind, "pos255"))
                if len(S.stages) > 1:
                    out.add(("err", kind, "stage2"))
            if m.k == 255 and isinstance(m.end, int):
                gb = [g for s, g, _ in S.checks if s == m.s][0]
                if rec + m.end > gb + STAGE - MARGIN and m.end - m.start <= 15:
                    out.add(("tail", m.end - m.start))
        for i, (s, L, n) in enumerate(S.windows):
            if n >= 126:
                ms = [m for m in S.members if m.s == s]
                odd = any(isinstance(m.end, int) and (m.end - m.start) % 2 for m in ms[:-1])
                out.add(("chain", n, "odd") if odd else ("chain", n))
                if n == 128 and ms[-1].end == s + L and L == WIN:
                    out.add(("chain", 128, "ends_at_L"))
        for s, gb, need in S.checks:
            if rec + need == gb + STAGE:
                out.add(("stage", "need_eq"))
        for s, gb, need in S.stages[1:]:
            prev = [c for c in S.checks if c[0] < s][-1][1]
            if rec + need == prev + STAGE + 1:
                out.add(("stage", "need_eq+1"))
            out.add(("restage_rec16", rec & 15))
            out.add(("restage_rec128", rec & 127))
        for a, e in S.groups:
            if e - a > 2 * STAGE:
                out.add(("group_skip", ">8K"))
            elif e - a > STAGE:
                out.add(("group_skip", ">4K"))
    if case.kind in (REGRESS, CLASSIFY) and len(sch) >= 2 and sch[1].checks and sch[0].stages:
        if (rec + sch[1].checks[0][0]) >= sch[0].stages[0][1] + STAGE:
            out.add(("result2_later_stage",))
    if case.kind == CLASSIFY and sch and sch[0].entries:
        off, ln = sch[0].entries[0]
        first = warp_entries(case.wire, off, off + ln, rec)
        if len(first.stages) > 1:
            out.add(("classes", len(first.entries), "restaged"))
    return out


# ---- the cases -----------------------------------------------------------------------------------------------------------------
@dataclass
class Case:
    name: str
    kind: object                 # REGRESS, CLASSIFY, or a list of kinds (MultiInference)
    wire: bytes
    rec: int = 0                 # the record's device address (its residues are what matter)
    targets: List[Tuple[str, int]] = field(default_factory=list)   # (field kind, record offset) of the placed fields
    member_bodies: Optional[List[Tuple[int, int]]] = None          # MultiInference: the member bodies the finder walks

    def schedules(self, rec):
        return [warp_entries(self.wire, lo, hi, rec) for lo, hi in (self.member_bodies or [])]


E00, U00, U3 = b"\x0a\x00", b"\x08\x00", b"\x10\x80\x01"   # an empty entry, an unknown 2-byte field, an unknown 3-byte field


def fill(n: int) -> bytes:
    """exactly n bytes of 2- and 3-byte fields (empty entries, unknown varints), n != 1"""
    assert n != 1
    out = b""
    if n % 2:
        out, n = U3, n - 3
    return out + (E00 + U00) * (n // 4) + (E00 if n % 4 else b"")


def pad(n: int) -> bytes:
    """exactly n bytes of unknown LEN fields (field 4), n != 1: few chain members"""
    assert n != 1
    out = b""
    while n:
        k = min(n, 129) if n - min(n, 129) != 1 else 128
        out += b"\x22" + bytes([k - 2]) + b"\x00" * (k - 2)
        n -= k
    return out


def _entry(v=1.5):
    return b"\x0a\x05\x0d" + f32(v)


# what a RegressionResult body may hold, by kind: (name, bytes)
def body_fields():
    out = [("entry_canon", _entry(2.5)), ("entry_empty", E00)]
    out += [(f"varint{n}", b"\x10" + varint(1, n - 1)) for n in range(1, 11)]
    out += [("i32", b"\x1d" + f32(7)), ("i64", b"\x19" + b"\x05" * 8)]
    out += [(f"len{n}", b"\x22" + varint(3, n - 1) + b"abc") for n in range(1, 6)]
    out += [(f"entry_tag{n}", X.long_tag(1, LEN, n) + b"\x05\x0d" + f32(3.5)) for n in range(2, 6)]
    out += [(f"entry_len{n}", b"\x0a" + varint(5, n - 1) + b"\x0d" + f32(4.5)) for n in range(2, 6)]
    out += [("entry_tag5_len5", X.long_tag(1, LEN, 5) + varint(5, 4) + b"\x0d" + f32(5.5))]   # 15 meaningful bytes
    out += [("group", b"\x4b\x08\x01\x4c")]
    out += [(f"group{d}", b"\x4b" * d + b"\x08\x01" + b"\x4c" * d) for d in range(1, 17)]
    return out


def bad_fields():
    """malformed fields of a body, by kind"""
    return [("len_past_hi", b"\x22\xff\x7f"), ("wt6", b"\x16\x00"), ("wt7", b"\x17\x00"), ("stray_egroup", b"\x14"),
            ("tag0", b"\x00\x00"), ("varint11", b"\x10" + b"\xff" * 10 + b"\x01"), ("tag6", X.long_tag(2, VARINT, 6) + b"\x01")]


def _regress(body: bytes, spec=True) -> Tuple[bytes, int]:
    """(response, record offset of the body)"""
    head = b"\x0a" + varint(len(body))
    tail = serialize(X.spec_nodes(version=3, signature=b"serving_default")) if spec else b""
    return head + body + tail, len(head)


def window_cases(rec=0) -> List[Case]:
    """Every body field kind starting at window-relative 253 to 256 and ending at s + 255 to s + 257 of the first window."""
    out = []
    for kind, fb in body_fields():
        w = len(fb)
        for at in sorted({253, 254, 255, 256} | {e - w for e in (255, 256, 257) if e - w >= 0}):
            if at == 1:
                continue
            body = fill(at) + fb + fill(600 - at - w if (600 - at - w) != 1 else 601 - at - w)
            wire, lo = _regress(body)
            out.append(Case(f"{kind}@{at}", REGRESS, wire, rec, [(kind, lo + at)]))
    return out


def chain_cases(rec=0) -> List[Case]:
    """Windows of 126, 127 and 128 two-byte members (empty entries and unknown varints), the 128-member chain ending exactly at
    the window's end, a 3-byte member that shifts the parity, and a response made of empty entries alone."""
    out = []
    for n in (126, 127, 128):
        for tail in (b"", _entry(6.5)):
            body = (E00 + U00) * (n // 2) + (E00 if n % 2 else b"")
            body = body[: 2 * n - 2] + (b"\x22\x00" if n < 128 else E00) + tail + fill(300)
            wire, lo = _regress(body)
            out.append(Case(f"chain{n}{'+entry' if tail else ''}", REGRESS, wire, rec))
        # a 3-byte member first: the chain runs over odd positions, and the last member ends one past the window
        body = U3 + (E00 + U00) * ((n - 1) // 2) + (E00 if (n - 1) % 2 else b"") + fill(300)
        wire, lo = _regress(body)
        out.append(Case(f"chain{n}_odd", REGRESS, wire, rec))
    body = E00 * 4000
    wire, _ = _regress(body, spec=False)
    out.append(Case("only_empty_entries", REGRESS, wire, rec))
    return out


def stage_cases(rec=0) -> List[Case]:
    """Bodies whose windows reach need == gb + 4096 (no restage) and gb + 4097 (restage), with a field of up to 15 meaningful
    bytes at the last window position before the stage ends; groups longer than 4 KB and 8 KB; a second result in a later
    stage."""
    out = []
    fields = dict(body_fields())
    for delta in (0, 1):
        for kind in ("entry_empty", "entry_canon", "i64", "varint10", "entry_tag5_len5"):
            fb = fields[kind]
            # the first window's exit is one LEN field of X bytes; then windows of 256 two-byte members: the 14th window
            # after it has need = s + 288 = gb + 4096 + delta when X = 480 + delta - a (a: the body's residue mod 16)
            lo = _regress(b"\0" * 6000)[1]      # every body here is 6000 bytes or longer: a 2-byte length
            a = (rec + lo) & 15
            x = 480 + delta - a
            first = b"\x22" + varint(x - 3) + b"\x00" * (x - 3)
            assert len(first) == x
            # windows 1..13 hold 128 members each; window 14 reaches position 255 with one 3-byte member, then the target
            body = first + fill(256 * 13) + U3 + fill(252) + fb + fill(400)
            wire, lo2 = _regress(body)
            assert lo2 == lo
            at = lo + x + 256 * 13 + 3 + 252
            out.append(Case(f"need_eq{'+1' if delta else ''}_{kind}", REGRESS, wire, rec, [(kind, at)]))
    for size in (5000, 9000):
        g = b"\x4b" + b"\x22" + varint(size) + b"\x00" * size + b"\x4c"
        body = fill(100) + g + fill(40) + _entry(7.5) + fill(30)
        wire, lo = _regress(body)
        out.append(Case(f"group_{size}", REGRESS, wire, rec, [("big_group", lo + 100)]))
    r1 = [(None, RAW, fill(5000)), (1, LEN, [(1, I32, f32(8.5))])]
    r2 = [(1, LEN, [(1, I32, f32(9.5))]), (None, RAW, fill(300)), (1, LEN, [])]
    wire = serialize([(1, LEN, r1), (15, LEN, b"\0" * 200)] + X.spec_nodes() + [(1, LEN, r2)])
    out.append(Case("result2", REGRESS, wire, rec))
    return out


def error_cases(rec=0) -> List[Case]:
    """A malformed field as the first window's exit, at window position 255, and in a second stage."""
    out = []
    for kind, fb in bad_fields():
        for name, at, total in (("w0", 40, 600), ("p255", 255, 600), ("stage2", 4700, 6000)):
            body = fill(at) + fb + b"\x22\x00" * 2
            if "len_past_hi" != kind:
                body += fill(total - len(body)) if total - len(body) != 1 else fill(total - len(body) + 1)
            wire, lo = _regress(body)
            out.append(Case(f"err_{kind}_{name}", REGRESS, wire, rec, [(kind, lo + at)]))
    return out


def group_depth_cases() -> List[Tuple[str, bytes, int]]:
    """(name, Regress wire, depth) with unknown groups nested `depth` deep inside the result body: the decode refuses more than
    16; the runtime accepts up to 99 there (100 with the message levels above)."""
    out = []
    for d in (16, 17, 40, 99, 100):
        g = b"\x4b" * d + b"\x08\x01" + b"\x4c" * d
        out.append((f"group_depth_{d}", _regress(fill(250) + g + _entry(1.25) + fill(10))[0], d))
    return out


def regress_grid(rec=0) -> List[Case]:
    return window_cases(rec) + chain_cases(rec) + stage_cases(rec) + error_cases(rec)


# ---- Classify --------------------------------------------------------------------------------------------------------------
def classify_response(examples, lead=b"", head_pad=0) -> bytes:
    """a ClassificationResponse: examples as for classification_nodes, an unknown top-level field of head_pad bytes first"""
    nodes = X.classification_nodes(examples)
    w = serialize(nodes)
    return (pad(head_pad) if head_pad else b"") + lead + w


def classify_groups():
    """{C: [(name, wire)]}: responses grouped by class count, so that every group decodes as one batch"""
    groups = {}

    def add(C, name, wire):
        groups.setdefault(C, []).append((name, wire))

    rng = np.random.default_rng(21)
    for C in (127, 128, 129, 1000):        # the first example's body crosses a stage
        labels = [f"c{k:04d}_{'l' * 36}".encode() for k in range(C)]   # ~50 bytes a class: past 4 KB
        for h in (0, 2, 131):
            ex = [[(lab, float(s)) for lab, s in zip(labels, rng.standard_normal(C).astype(np.float32))] for _ in range(3)]
            add(C, f"classes{C}_pad{h}", classify_response(ex, head_pad=h))
    for C in (31, 32, 33, 64):
        labels = [f"L{k}".encode() for k in range(C)]
        for n in (1, 5):
            add(C, f"lanes{C}_{n}", classify_response([[(lab, float(k)) for k, lab in enumerate(labels)]] * n))
    # labels of 0 to 300 bytes across the emit cursor's 128-byte lines, a multi-byte character split across a line
    for L in (0, 1, 63, 127, 128, 129, 255, 300):
        for h in (0, 2, 5, 61, 124):
            lab = (b"x" * L)
            add(2, f"label{L}_pad{h}", classify_response([[(lab, 1.0), ("é€😀".encode() * 3, 2.0)]] * 3, head_pad=h))
    for h in range(0, 130, 3):
        add(2, f"utf8_split_pad{h}", classify_response([[(("€" * 50 + "😀" * 20).encode(), 0.5), (b"b", -1.0)]] * 2, head_pad=h))
    # a row served by a later CTA than the first whose labels differ from the first example's in their last byte only
    ex = [[(b"label_aaaa", 1.0), (b"label_bbbb", 2.0)]] * 700
    ex[600] = [(b"label_aaaa", 1.0), (b"label_bbbc", 2.0)]
    add(2, "late_row_last_byte", classify_response(ex))
    add(2, "late_row_same", classify_response([[(b"label_aaaa", 1.0), (b"label_bbbb", 2.0)]] * 700))
    return groups


# ---- Regress emit: entries the cursor walks --------------------------------------------------------------------------------
def emit_cases() -> List[Tuple[str, bytes]]:
    """Non-canonical Regression entries (the emit walks them through its two-line cursor), each across a 128-byte line"""
    ents = [("padded_tag", X.long_tag(1, I32, 3) + f32(1.75)), ("two_values", b"\x0d" + f32(1.0) + b"\x0d" + f32(-2.0)),
            ("unknown_first", b"\x10\x05\x22\x03abc\x0d" + f32(3.0)), ("five_not_0d", b"\x10\x80\x80\x80\x01"),
            ("five_i32_unknown", b"\x15" + f32(9.0))]
    out = []
    for name, e in ents:
        for at in range(100, 130, 1):
            body = pad(at) + b"\x0a" + varint(len(e)) + e + fill(20)
            out.append((f"{name}@{at}", _regress(body)[0]))
    return out


# ---- MultiInference ----------------------------------------------------------------------------------------------------------
def multi_cases(rec=0) -> List[Case]:
    """The window, stage and tag cases inside a task's member body; 1 to 4 tasks of mixed kinds; a oneof switch whose cleared
    member straddles a window edge; repeated occurrences of the surviving member in different stages."""
    C, R = CLASSIFY, REGRESS
    ex = [[(b"pos", 0.25), (b"neg", 0.75)]] * 3
    small = {C: M.result(M.CLS, M.cls_body(ex)), R: M.result(M.REG, M.reg_body([1.0, -2.0]))}
    out = []
    grid = [c for c in regress_grid(rec) if not c.name.startswith("result2")]
    task_sets = ([R], [C, R], [R, C, R], [C, R, R, C])
    for i, case in enumerate(grid[::3]):
        results_ = results(case.wire)
        lo, hi = results_[0]
        body = case.wire[lo:hi]
        kinds = task_sets[i % 4]
        t = kinds.index(R)
        nodes = [small[k] for k in kinds]
        nodes[t] = (1, LEN, M.spec(version=1) + [(M.REG, LEN, [(None, RAW, body)])])
        wire = serialize(nodes)
        off = wire.find(body)
        shift = off - lo
        out.append(Case("mi_" + case.name, kinds, wire, rec, [(k, a + shift) for k, a in case.targets], [(off, off + len(body))]))
    # the oneof: a cleared classification member straddling 256, then the surviving regression member
    for cl in (240, 250, 253, 256, 300):
        cleared = (M.CLS, LEN, [(None, RAW, fill(cl))])
        keep = (M.REG, LEN, [(None, RAW, fill(200)), (1, LEN, [(1, I32, f32(2.25))])])
        wire = serialize([(1, LEN, M.spec() + [cleared, keep]), small[C]])
        out.append(Case(f"mi_oneof_cleared{cl}", [R, C], wire, rec))
        wire = serialize([(1, LEN, [(M.REG, LEN, [(None, RAW, fill(cl))]), (M.CLS, LEN, M.cls_body(ex))])])
        out.append(Case(f"mi_oneof_to_cls{cl}", [C], wire, rec))
    # the surviving member again, in a later stage
    r = (1, LEN, [(M.REG, LEN, [(None, RAW, fill(5000)), (1, LEN, [(1, I32, f32(3.25))])]), (20, LEN, b"\0" * 300),
                  (M.REG, LEN, [(1, LEN, [(1, I32, f32(4.25))]), (None, RAW, fill(4500))]), (M.REG, LEN, [(1, LEN, [])])])
    out.append(Case("mi_member_stages", [R, C], serialize([r, small[C]]), rec))
    for name, kinds, wire in M.long_tag_cases():
        out.append(Case("mi_" + name, kinds, wire, rec))
    return out


def member_bodies(wire: bytes, kinds) -> Optional[List[Tuple[int, int]]]:
    """[(lo, hi)] of every member body the finder walks, by a serial walk of the response (None: malformed top level)"""
    rs = results(wire)
    if rs is None:
        return None
    out = []
    for t, (lo, hi) in enumerate(rs[: len(kinds)]):
        member = M.CLS if kinds[t] == CLASSIFY else M.REG
        sub = wire[:hi]
        p, last = lo, None
        bodies = []
        while p < hi:
            tg = _tag_at(sub, p, hi)
            if tg is None:
                return None
            if tg[0] >> 3 in (M.CLS, M.REG) and tg[0] & 7 == LEN:
                v = _varint_at(sub, tg[1], hi)
                if v is None:
                    return None
                if tg[0] >> 3 != last:
                    bodies, last = [], tg[0] >> 3
                bodies.append((v[1], v[1] + v[0]))
                p = v[1] + v[0]
                continue
            e = _skip_any(sub, p, hi)
            if e == ERR:
                return None
            p = e
        if last == member:
            out += bodies
    return out


def as_f32(bits) -> float:
    return struct.unpack("<f", struct.pack("<I", bits))[0]
