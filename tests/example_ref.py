"""Reference of the tf.Example request encode (csrc/example_kernels.cuh, planned by csrc/example_host.inc): the exact bytes of
a Classify / Regress or Predict request written with numpy from the proto field numbers, and a model of the kernels' geometry
- the host plan, every emit batch, the scan's carry rounds, the frame kernel's lane rounds and the nested lengths - computed
from the plan and the real example sizes.

The byte reference uses neither protobuf nor the codec: it scales to millions of examples and, through ``examples_chunk``, to
gigabyte requests made of a few distinct examples.  tests/test_example_reference_cpu.py pins it byte for byte against the
protobuf runtime and pins the model against the sources; tests/test_example_edges_gpu.py compares the device with it and asks
the model which edges each case reached.  The kernels' constants are read from the sources, so the model cannot drift silently.

Wire, as the runtime serialises it with ``deterministic=True``:
  example      {0A | 42} vi(X) 0A vi(F) entry...              X = Features message, F = the map entries
  entry        0A vi(entry) 0A vi(klen) key 12 vi(feature) {12 float_list | 1A int64_list} vi(list) [0A vi(P) payload]
               (an empty list: vi(list) = 00 and nothing behind it), or for a bytes column (BytesColumn)
               0A vi(entry) 0A vi(klen) key 12 vi(feature) 0A vi(P) {0A vi(len) bytes}...   (P = 0 for a row of no strings)
  Classify     spec 12 vi(outer) 0A vi(inner) examples        outer = Input, inner = ExampleList
  Predict      spec 12 vi(outer) 0A vi(klen) key 12 vi(inner) 08 07 12 vi(shape) shape examples
  with context spec 12 vi(outer) 12 vi(elwc) elwc              elwc = examples (tag 0A) 12 vi(X) context
               (Predict: the map entry's TensorProto is DT_STRING [1] with the elwc as its one string_val)
"""
import functools
import os
import re

import numpy as np

from min_tfs_client.codec import BytesColumn, RaggedColumn

_CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "min-tfs-client_b200", "csrc")


def _source(fname):
    with open(os.path.join(_CSRC, fname)) as f:
        return f.read()


def _const(fname, name):
    m = re.search(r"constexpr\s+uint32_t\s+%s\s*=\s*(\w+)u?\s*;" % name, _source(fname))
    assert m, (fname, name)
    v = m.group(1)
    return int(v) if v.isdigit() else _const(fname, v)


K_STAGE = _const("plan.h", "kExStage")              # bytes of the emit kernel's shared-memory image
K_EMIT_THREADS = _const("plan.h", "kExEmitThreads")
K_PLAN_THREADS = _const("plan.h", "kConcatPlanThreads")
K_TILE = _const("plan.h", "kExTile")                 # examples per count / scan tile, and tiles per carry round of the scan
K_FRAME_LANES = 32                                   # the frame kernel sums tile sums one warp at a time
K_CHUNK = 32                                         # ex_write_example: features per warp pass
PROTO_LIMIT = 0x7FFFFFFF


# ---- varints ---------------------------------------------------------------------------------------------------------------
def vlen(v):
    """bytes of the varint of every element of v (uint64 view)"""
    v = np.asarray(v).astype(np.uint64, copy=False)
    n = np.ones(v.shape, np.int64)
    for k in range(1, 10):
        n += v >= np.uint64(1 << (7 * k))
    return n


def vi(v: int) -> bytes:
    out = bytearray()
    v &= (1 << 64) - 1
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def varints(v):
    """(bytes of each varint, the varints of v back to back)"""
    v = np.asarray(v).astype(np.uint64, copy=False).ravel()
    if len(v) > 1 << 22:        # bounded temporaries
        parts = [varints(v[a: a + (1 << 22)]) for a in range(0, len(v), 1 << 22)]
        return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])
    n = vlen(v)
    K = int(n.max()) if len(v) else 1
    k = np.arange(K, dtype=np.uint64)
    b = ((v[:, None] >> (np.uint64(7) * k)) & np.uint64(0x7F)).astype(np.uint8)
    b |= np.where(k[None, :].astype(np.int64) < (n - 1)[:, None], 0x80, 0).astype(np.uint8)
    return n, b[np.arange(K)[None, :] < n[:, None]]


# ---- pieces: per-example byte strings, (lengths[n], bytes back to back) ----------------------------------------------------
def _const_piece(n, c: bytes):
    return np.full(n, len(c), np.int64), np.tile(np.frombuffer(c, np.uint8), n)


def _join(pieces):
    """per example, the pieces one after the other"""
    if len(pieces[0][0]) == 1:       # one example: no scatter (requests of hundreds of megabytes)
        return sum(p[0] for p in pieces), np.concatenate([p[1] for p in pieces])
    lens = np.stack([p[0] for p in pieces], 1)
    tot = lens.sum(1)
    out = np.empty(int(tot.sum()), np.uint8)
    start = np.cumsum(tot) - tot + (np.cumsum(lens, 1) - lens).T
    for j, (ln, flat) in enumerate(pieces):
        if len(flat):
            out[np.repeat(start[j] - (np.cumsum(ln) - ln), ln) + np.arange(len(flat))] = flat
    return tot, out


def _where(mask, piece):
    """the piece of every example where mask holds (piece covers those examples only), empty elsewhere"""
    ln = np.zeros(len(mask), np.int64)
    ln[mask] = piece[0]
    return ln, piece[1]


# ---- columns ---------------------------------------------------------------------------------------------------------------
def _f32_bits(a):
    """float32 bits of a float array as examples_from_input_dict stores them: astype(float32), then the trip through a Python
    float quiets every NaN"""
    with np.errstate(all="ignore"):
        b = np.asarray(a).astype(np.float32).view(np.uint32)
    nan = (b & 0x7FFFFFFF) > 0x7F800000
    return np.where(nan, b | 0x00400000, b).astype(np.uint32)


def _i64(a):
    a = np.asarray(a)
    if a.dtype == np.bool_:
        return (a.view(np.uint8) != 0).astype(np.uint64)     # any nonzero byte is True
    return a.astype(np.int64).view(np.uint64)


class Col:
    """one column: key, float (float_list) or not (int64_list), each example's element count and its elements back to back"""

    def __init__(self, key, value, n, values=True):
        self.key = key.encode("utf-8") if isinstance(key, str) else bytes(key)
        self.ragged = isinstance(value, RaggedColumn)
        inner = value.values if self.ragged else value
        self.is_bytes = isinstance(inner, BytesColumn)
        if self.is_bytes:
            self._bytes(inner, value.lengths if self.ragged else None, n, values)
            return
        a = np.asarray(value.values) if self.ragged else np.asarray(value)
        self.is_float = a.dtype.kind == "f"
        self.dtype = a.dtype
        if self.ragged:
            unit = int(np.prod(a.shape[2:], dtype=np.int64))
            self.row_elems = a.shape[1] * unit
            self.ne = np.clip(np.asarray(value.lengths).astype(np.int64), 0, a.shape[1]) * unit
        elif a.ndim == 0:
            self.row_elems = 1
            self.ne = np.ones(n, np.int64)
        else:
            self.row_elems = int(np.prod(a.shape[1:], dtype=np.int64))
            self.ne = np.full(n, self.row_elems, np.int64)
        if not values:
            return
        if self.ragged:
            elems = a.reshape(n, -1)[np.arange(self.row_elems)[None, :] < self.ne[:, None]]
        else:
            elems = np.repeat(a.reshape(1), n) if a.ndim == 0 else a.reshape(-1)
        if self.is_float:
            self.payload = _f32_bits(elems).view(np.uint8)
            self.P = 4 * self.ne
        else:
            ln, self.payload = varints(_i64(elems))
            cs = np.concatenate([[0], np.cumsum(ln)])
            ends = np.cumsum(self.ne)
            self.P = cs[ends] - cs[ends - self.ne]

    def _bytes(self, col, lengths, n, values):
        """a bytes_list column (BytesColumn, or a RaggedColumn of one): each example's strings, 0A vi(len) bytes each"""
        self.is_float, self.dtype = False, np.dtype(np.uint8)
        shape = tuple(col.shape)
        self.row_elems = int(np.prod(shape[1:], dtype=np.int64)) if shape else 1
        if lengths is not None:
            unit = int(np.prod(shape[2:], dtype=np.int64))
            self.ne = np.clip(np.asarray(lengths).astype(np.int64), 0, shape[1]) * unit
        else:
            self.ne = np.full(n, self.row_elems, np.int64)
        self.data_len, self.broadcast = int(col.data_len), not shape      # what the host plan sizes the column by
        if not values:
            return
        data, off = np.asarray(col.data), np.asarray(col.offsets).astype(np.int64)
        stride = 0 if not shape else self.row_elems
        cells = np.arange(self.row_elems)[None, :]
        idx = (np.arange(n)[:, None] * stride + cells)[cells < self.ne[:, None]]      # the strings of every row, row after row
        lens = off[idx + 1] - off[idx]
        out_start = np.cumsum(lens) - lens
        strings = data[np.repeat(off[idx] - out_start, lens) + np.arange(int(lens.sum()))]
        if len(idx):
            sz, self.payload = _join([_const_piece(len(idx), b"\x0a"), varints(lens), (lens, strings)])
        else:
            sz, self.payload = np.zeros(0, np.int64), np.zeros(0, np.uint8)
        ends = np.cumsum(self.ne)
        cs = np.concatenate([[0], np.cumsum(sz)])
        self.P = cs[ends] - cs[ends - self.ne]


def upb_order(keys):
    """the map order of the deterministic runtime: bytewise on the common prefix, the longer key first on a tie"""
    def cmp(a, b):
        m = min(len(a), len(b))
        if a[:m] != b[:m]:
            return -1 if a[:m] < b[:m] else 1
        return len(b) - len(a)
    return sorted(range(len(keys)), key=functools.cmp_to_key(lambda i, j: cmp(keys[i], keys[j]) or i - j))


def _rows(v):
    """example count of a column; None for a 0-d (broadcast) one"""
    if isinstance(v, RaggedColumn):
        v = v.values
    shape = tuple(v.shape) if isinstance(v, BytesColumn) else np.shape(v)
    return shape[0] if shape else None


def n_examples(d):
    rows = {_rows(v) for v in d.values()} - {None}
    assert len(rows) <= 1
    return rows.pop() if rows else (1 if d else 0)


def columns(d, order="deterministic", values=True):
    """(n, the columns of input dict d in wire order; without values: keys, kinds and element counts only)"""
    n = n_examples(d)
    cols = [Col(k, v, n, values) for k, v in d.items()]
    if order != "given":
        cols = [cols[i] for i in upb_order([c.key for c in cols])]
    return n, cols


def nested(cols, n):
    """every nested length of every example: P, list, feature, entry (per column, [n_cols, n]), F, X and S ([n])"""
    P = np.stack([c.P for c in cols]) if cols else np.zeros((0, n), np.int64)
    klen = np.array([len(c.key) for c in cols], np.int64)[:, None]
    is_bytes = np.array([c.is_bytes for c in cols], bool)[:, None]
    lst = np.where(is_bytes, P, np.where(P > 0, 1 + vlen(P) + P, 0))      # a BytesList is its values, unpacked
    feature = 1 + vlen(lst) + lst
    entry = 1 + vlen(klen) + klen + 1 + vlen(feature) + feature
    F = (1 + vlen(entry) + entry).sum(0)
    X = 1 + vlen(F) + F
    return {"P": P, "list": lst, "feature": feature, "entry": entry, "F": F, "X": X, "S": 1 + vlen(X) + X}


def example_bytes(d, order="deterministic", tag=0x0A):
    """(byte length of every example with its tag, every example's bytes back to back)"""
    n, cols = columns(d, order)
    if n == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.uint8)
    L = nested(cols, n)
    pieces = [_const_piece(n, bytes([tag])), varints(L["X"]), _const_piece(n, b"\x0a"), varints(L["F"])]
    for k, c in enumerate(cols):
        has = c.P > 0
        pieces += [_const_piece(n, b"\x0a"), varints(L["entry"][k]), _const_piece(n, b"\x0a" + vi(len(c.key)) + c.key + b"\x12"),
                   varints(L["feature"][k]), _const_piece(n, b"\x0a" if c.is_bytes else b"\x12" if c.is_float else b"\x1a"),
                   varints(L["list"][k])]
        if not c.is_bytes:
            pieces.append(_where(has, _join([_const_piece(int(has.sum()), b"\x0a"), varints(c.P[has])])))
        pieces.append((c.P, c.payload))
    S, flat = _join(pieces)
    assert (S == L["S"]).all()
    return S, flat


# ---- request framing -------------------------------------------------------------------------------------------------------
def model_spec(name, version) -> bytes:
    nb = name.encode("utf-8") if isinstance(name, str) else bytes(name)
    body = (b"\x0a" + vi(len(nb)) + nb) if nb else b""
    if version is not None:
        v = (b"\x08" + vi(version)) if version else b""
        body += b"\x12" + vi(len(v)) + v
    return b"\x0a" + vi(len(body)) + body


def predict_head(n) -> bytes:
    """TensorProto fields in front of string_val: dtype DT_STRING, tensor_shape [n]"""
    dim = (b"\x08" + vi(n)) if n else b""
    shape = b"\x12" + vi(len(dim)) + dim
    return b"\x08\x07\x12" + vi(len(shape)) + shape


def framing(spec, n, el, key=None):
    """(mid, head, inner, outer, msg) of a request whose examples take el bytes (key: the Predict input key, None: example_list)"""
    kb = None if key is None else (key.encode("utf-8") if isinstance(key, str) else bytes(key))
    mid = b"" if kb is None else b"\x0a" + vi(len(kb)) + kb
    head = b"" if kb is None else predict_head(n)
    inner = len(head) + el
    outer = len(mid) + 1 + len(vi(inner)) + inner
    return mid, head, inner, outer, len(spec) + 1 + len(vi(outer)) + outer


def prefix(name, version, n, el, key=None, grpc=False) -> bytes:
    """the bytes in front of the examples"""
    spec = model_spec(name, version)
    mid, head, inner, outer, msg = framing(spec, n, el, key)
    g = (b"\x00" + msg.to_bytes(4, "big")) if grpc else b""
    return g + spec + b"\x12" + vi(outer) + mid + (b"\x0a" if key is None else b"\x12") + vi(inner) + head


def _one_example(v):
    """a context column (the one example's row, as requests.py takes it) as a column of one example"""
    if isinstance(v, BytesColumn):
        return v if not v.shape else BytesColumn(v.data, v.offsets, (1,) + tuple(v.shape))
    a = np.asarray(v)
    return a if a.ndim == 0 else a[None]


def context_bytes(context, order="deterministic") -> bytes:
    """the ExampleListWithContext.context field (tag 12) of a context dict; 12 00 for an empty one"""
    if not context:
        return b"\x12\x00"
    return example_bytes({k: _one_example(v) for k, v in context.items()}, order, 0x12)[1].tobytes()


def request_bytes(name, version, d, key=None, grpc=False, order="deterministic", context=None) -> bytes:
    """the whole request: a ClassificationRequest / RegressionRequest (key None) or a PredictRequest whose input `key` holds
    the examples; with grpc, behind gRPC's five-byte length-prefixed-message header.  With a context (a dict, {} included) the
    examples and the context form an ExampleListWithContext: Input field 2, or the one string_val of the Predict input"""
    if context is None:
        S, flat = example_bytes(d, order, 0x0A if key is None else 0x42)
        return prefix(name, version, len(S), int(S.sum()), key, grpc) + flat.tobytes()
    elwc = example_bytes(d, order, 0x0A)[1].tobytes() + context_bytes(context, order)
    spec = model_spec(name, version)
    if key is None:                                     # Input { example_list_with_context = 2 }
        outer = b"\x12" + vi(len(elwc)) + elwc
        msg = spec + b"\x12" + vi(len(outer)) + outer
    else:                                               # inputs[key] = DT_STRING [1] holding the serialized ELWC
        kb = key.encode("utf-8") if isinstance(key, str) else bytes(key)
        tp = predict_head(1) + b"\x42" + vi(len(elwc)) + elwc
        ent = b"\x0a" + vi(len(kb)) + kb + b"\x12" + vi(len(tp)) + tp
        msg = spec + b"\x12" + vi(len(ent)) + ent
    return ((b"\x00" + len(msg).to_bytes(4, "big")) if grpc else b"") + msg


def examples_chunk(ex, pattern, i0, i1):
    """bytes of examples [i0, i1) of a request made of a few distinct examples: example i is ex[pattern[i]] (ex: their bytes,
    from example_bytes); runs of one example are tiled, not looped over"""
    p = pattern[i0:i1]
    cut = np.flatnonzero(np.diff(p)) + 1
    starts, ends = np.concatenate([[0], cut]), np.concatenate([cut, [len(p)]])
    return np.concatenate([np.tile(ex[p[a]], b - a) for a, b in zip(starts, ends)]) if len(p) else np.zeros(0, np.uint8)


# ---- geometry model --------------------------------------------------------------------------------------------------------
def _entry_len(P, klen):
    lst = 1 + len(vi(P)) + P if P else 0
    feature = 1 + len(vi(lst)) + lst
    entry = 1 + len(vi(klen)) + klen + 1 + len(vi(feature)) + feature
    return 1 + len(vi(entry)) + entry


def _bytes_entry_len(P, klen):
    feature = 1 + len(vi(P)) + P
    entry = 1 + len(vi(klen)) + klen + 1 + len(vi(feature)) + feature
    return 1 + len(vi(entry)) + entry


def _example_len(F):
    x = 1 + len(vi(F)) + F
    return 1 + len(vi(x)) + x


class ReqPlan:
    """what example_host.inc plans for one request, from its columns alone (no values)"""

    def __init__(self, name, version, d, key=None, grpc=False):
        self.n, cols = columns(d, values=False)
        self.n_feat = len(cols)
        self.has_int = any(not c.is_float and not c.is_bytes for c in cols)
        self.has_bytes = any(c.is_bytes for c in cols)
        self.counted = self.has_int or self.has_bytes or any(c.ragged for c in cols)
        num = [c for c in cols if not c.is_bytes]
        f_max = sum(_entry_len((4 if c.is_float else 10) * c.row_elems, len(c.key)) for c in num)
        f_min = sum(_entry_len((4 if c.is_float else 1) * c.row_elems, len(c.key)) for c in num)
        # a bytes column: no strings plus 27 bytes of length varints at most, two bytes per string at least
        f_max += sum(_bytes_entry_len(0, len(c.key)) + 27 for c in cols if c.is_bytes)
        f_min += sum(_bytes_entry_len(2 * c.row_elems, len(c.key)) for c in cols if c.is_bytes)
        self.ex_max, self.ex_min = _example_len(f_max), _example_len(f_min)
        self.str_bound, self.ex_expect = 0, self.ex_max
        if self.has_bytes:        # ex_layout: the strings' bound, and the planner's guess of an example's size for the spans
            self.ex_max += 18
            self.ex_expect = self.ex_max
            for c in cols:
                if c.is_bytes:
                    D, R = min(c.data_len, PROTO_LIMIT), c.row_elems
                    self.str_bound += self.n * R * 11 + (self.n * D if c.broadcast else D)
                    self.ex_expect += 2 * R + (D if c.broadcast or not self.n else D // self.n)
        self.spec = model_spec(name, version)
        mid, head, _, _, _ = framing(self.spec, self.n, 0, key)
        self.grpc, self.predict = grpc, key is not None
        self.prefix_max = (5 if grpc else 0) + len(self.spec) + len(mid) + len(head) + 22
        self.per = max(1, K_STAGE // self.ex_expect)
        self.spans = [(e0, min(e0 + self.per, self.n)) for e0 in range(0, self.n, self.per)]


def plan(reqs):
    """the host plan of one call: reqs = [ReqPlan]; sets slot_off, anchor, slot_end, first_tile and n_tiles on each"""
    cursor = tiles = 0
    for q in reqs:
        q.slot_off = (cursor + 255) & ~255
        q.anchor = (q.slot_off + q.prefix_max + 15) & ~15
        q.slot_end = cursor = q.anchor + q.n * q.ex_max + q.str_bound
        q.first_tile = tiles
        q.n_tiles = -(-q.n // K_TILE) if q.counted else 0
        tiles += q.n_tiles
    return cursor


def emit(q, sizes):
    """ex_emit over every span of request q whose examples take `sizes` bytes: a dict of what the loop did
      batches       (ws, lo, j, be - ws, carried) of every batch that wrote examples into the image
      full          batches whose examples end exactly at the end of the image
      carried       partial-vector lengths moved to the front of the image
      multi         spans that took more than one batch
      in_place      (start % 16, end % 16, bytes flushed in front) of every example written in place
      stores        every [lo, hi) the CTAs store, for the coverage check
      span_phases   the arena phases mod 16 at which spans start
      sharers       most spans that store into one 16-byte vector"""
    ends = q.anchor + np.cumsum(sizes)
    starts = ends - sizes
    out = {"batches": [], "full": 0, "carried": set(), "multi": 0, "in_place": [], "stores": [], "span_phases": set(), "sharers": 0}
    for e0, e1 in q.spans:
        lo = int(starts[e0])
        ws, i, nb = lo & ~15, e0, 0
        out["span_phases"].add(lo & 15)
        while i < e1:
            j = i + int(np.searchsorted(ends[i:e1], ws + K_STAGE, side="right"))
            if j > i:
                nb += 1
                be = int(ends[j - 1])
                cut = be & ~15
                out["full"] += be - ws == K_STAGE
                carried = be - cut if cut > ws else None
                out["batches"].append((ws, lo, j, be - ws, carried))
                if cut > ws:
                    out["stores"].append((lo, cut))
                    out["carried"].add(be - cut)
                    ws = lo = cut
                i = j
            else:
                s, e = int(starts[i]), int(ends[i])
                out["stores"] += [(lo, s), (s, e)]
                out["in_place"].append((s & 15, e & 15, s - lo))
                lo, ws, i = e, e & ~15, i + 1
        out["stores"].append((lo, int(ends[e1 - 1])))
        out["multi"] += nb > 1
    # span s stores [starts[e0], ends[e1 - 1]): the spans after it that start inside its last vector share that vector
    sp = [(int(starts[e0]), int(ends[e1 - 1])) for e0, e1 in q.spans if ends[e1 - 1] > starts[e0]]
    if sp:
        first_vec = np.array([a >> 4 for a, _ in sp])
        last_vec = np.array([(b - 1) >> 4 for _, b in sp])
        out["sharers"] = int((np.searchsorted(first_vec, last_vec, side="right") - np.arange(len(sp))).max())
    return out


def covers_once(q, sizes, stores):
    """do the stores cover [anchor, anchor + total) exactly once?"""
    r = sorted((a, b) for a, b in stores if b > a)
    at = q.anchor
    for a, b in r:
        if a != at:
            return False
        at = b
    return at == q.anchor + int(np.sum(sizes))


def scan_rounds(q):
    """the scan kernel's carry rounds of every tile of q: tile t sums the tiles in front of it kExTile at a time"""
    return [-(-t // K_TILE) for t in range(q.n_tiles)]


def frame_rounds(q):
    """the frame kernel's lane rounds over q's tile sums"""
    return -(-q.n_tiles // K_FRAME_LANES)


def chunks(q):
    """ex_write_example's warp passes over q's features"""
    return -(-q.n_feat // K_CHUNK)


def request_lengths(q, el, key=None):
    """the request-level nested lengths: inner (example_list or TensorProto), outer (Input or map entry) and msg"""
    _, _, inner, outer, msg = framing(q.spec, q.n, el, key)
    return {"inner": inner, "outer": outer, "msg": msg}


# ---- edge cases: inputs that put the encode on a chosen edge (small versions run on the CPU against the runtime) -------------
KINDS = ("f32", "int", "ragged_int", "zero_d", "zero_width", "ragged_f32")


def chunk_case(n_feat, rot, n=40, seed=0):
    """n_feat features whose kinds cycle through KINDS from `rot` on, keys in index order: over the rotations, lane 31 and lane 0
    of every chunk boundary hold every kind, and integer columns sit in every chunk"""
    rng = np.random.default_rng(seed)
    d = {}
    for k in range(n_feat):
        kind = KINDS[(k + rot) % len(KINDS)]
        lengths = rng.integers(0, 5, n)
        lengths[::3] = 0                                  # empty payloads (P = 0) in every column that can have one
        if kind == "f32":
            v = rng.standard_normal((n, 2)).astype(np.float32)
        elif kind == "int":
            v = rng.integers(-(1 << 40), 1 << 40, (n, 3)) >> rng.integers(0, 40, (n, 3))
        elif kind == "ragged_int":
            v = RaggedColumn(rng.integers(-300, 300, (n, 4)).astype(np.int16), lengths)
        elif kind == "zero_d":
            v = np.float64(k)
        elif kind == "zero_width":
            v = np.zeros((n, 0), np.float32)
        else:
            v = RaggedColumn(rng.standard_normal((n, 4)).astype(np.float32), lengths)
        d["f%03d" % k] = v
    return d


def _lens_ab(L, m):
    """nested lengths of an example of two int64_list columns "a" and "b" of L and m one-byte varints"""
    out = {}
    F = 0
    for key, P in (("a", L), ("b", m)):
        lst = 1 + len(vi(P)) + P if P else 0
        feature = 1 + len(vi(lst)) + lst
        entry = 3 + 1 + len(vi(feature)) + feature
        if key == "a":
            out.update(P=P, list=lst, feature=feature, entry=entry)
        F += 1 + len(vi(entry)) + entry
    out.update(F=F, X=1 + len(vi(F)) + F)
    return out


NESTED = ("P", "list", "feature", "entry", "F", "X")


def nested_case(targets):
    """one example per (quantity, value) of targets, whose `quantity` (a name of NESTED) is exactly `value`: ragged columns "a"
    and "b" of ones, cut to the lengths that give it.  Returns (input dict, [(quantity, value)])"""
    want, La, Lb = [], [], []
    for q in NESTED:
        for t in targets:
            hit = next(((L, m) for L in range(max(0, t - 40), t + 1) for m in range(4) if _lens_ab(L, m)[q] == t), None)
            assert hit, (q, t)
            want.append((q, t))
            La.append(hit[0])
            Lb.append(hit[1])
    n, M = len(want), max(La)
    d = {"a": RaggedColumn(np.ones((n, M), np.int8), np.array(La)), "b": RaggedColumn(np.ones((n, 3), np.int8), np.array(Lb))}
    return d, want


def fixed_size(S, n, seed=0):
    """a float-only input dict whose examples take exactly S bytes each (tag included)"""
    for w in range(max(0, (S - 30) // 4), S // 4 + 1):
        for klen in range(1, 20):
            if _example_len(_entry_len(4 * w, klen)) == S:
                return {"k" * klen: np.random.default_rng(seed).standard_normal((n, w)).astype(np.float32)}
    raise AssertionError(S)


def request_case(quantity, target, key=None):
    """(name, input dict) of one float-only example whose request-level `quantity` (inner, outer) is exactly target"""
    for w in range(max(0, (target - 80) // 4), target // 4 + 1):
        for klen in range(1, 40):
            el = _example_len(_entry_len(4 * w, klen))
            _, _, inner, outer, _ = framing(model_spec("m", 1), 1, el, key)
            if {"inner": inner, "outer": outer}[quantity] == target:
                return {"k" * klen: np.arange(w, dtype=np.float32).reshape(1, w)}
    raise AssertionError((quantity, target))


def counted_case(n, seed=0):
    """a counted request of n examples whose sizes vary"""
    rng = np.random.default_rng(seed)
    return {"i": rng.integers(0, 1 << 35, (n, 2)) >> rng.integers(0, 35, (n, 2)), "x": rng.standard_normal((n, 1)).astype(np.float32)}
