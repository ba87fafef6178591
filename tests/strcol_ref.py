"""Reference and geometry model of the routes over offset-indexed byte columns (csrc/strcol.h and its users): the padded
DT_STRING request encode (unpad_str_*_kernel), the concatenated and padded DT_STRING response decodes (str_* / pad_str_*_kernel)
and the tf.Example bytes_list encode (ex_write_bytes; its bytes come from tests/example_ref.py, which takes BytesColumn features).

The byte reference is numpy over the field numbers, without protobuf, so cases of millions of strings made of a few distinct ones
stay fast; tests/test_strcol_reference_cpu.py pins it against the protobuf runtime and the protobuf-backed definitions
(string_responses.reference, padded_string_decode_ref.reference).  The geometry model answers, from the sizes and addresses the
kernels see, which edge a case reached; tests/test_strcol_edges_gpu.py asserts through it.  The kernels' constants are read from
the sources, so a retuned threshold moves the edges instead of silently skipping them.

Wire pieces:
  string value       tag vi(len) bytes                  tag 42 (TensorProto.string_val) or 0A (BytesList.value)
  TensorProto        08 07 12 vi(shape) {12 vi(dim) [08 vi(size)]}... 42 vi(len) bytes...
  PredictRequest     0A vi(spec) spec {12 vi(entry) 0A vi(klen) key 12 vi(tp) tp}...      (map entries in key order)
"""
import re

import numpy as np

import example_ref as E

vi, varints = E.vi, E.varints


def _const(fname, name):
    m = re.search(r"constexpr\s+uint(?:32|64)_t\s+%s\s*=\s*(\w+?)(?:u|ull)?\s*;" % name, E._source(fname))
    assert m, (fname, name)
    v = m.group(1)
    return int(v) if v.isdigit() else _const(fname, v)


def _line_bytes():
    """the cursor's line: cur_open rounds the record's address down to it"""
    m = re.search(r"\(uintptr_t\)rec\s*&\s*~\(uintptr_t\)(\d+)", E._source("walker.h"))
    assert m
    return int(m.group(1)) + 1


K_LANE = _const("strcol.h", "kStrLaneCopy")                 # at most this long: a lane's own copy; longer: the warp's
K_BLOCK = _const("unpad_kernels.cuh", "kUnpadStrBlockCopy")  # padded encode only: longer than this goes to the CTA
K_CHUNK = _const("plan.h", "kStrChunk")                     # strings per copy chunk of the concatenated decode
K_STR_THREADS = _const("plan.h", "kStrThreads")             # threads per CTA of the decodes' index / copy / fix kernels
K_VAR_THREADS = _const("plan.h", "kVarThreads")             # strings per tile of the padded encode
K_GROUP_TILES = _const("plan.h", "kVarGroupTiles")          # tiles per counter group (prefix_share)
K_STAGE = E.K_STAGE
LINE = _line_bytes()
WARP = 32


# ---- bytes -----------------------------------------------------------------------------------------------------------------
def lens_of(strs):
    return np.array([len(s) for s in strs], np.int64)


def flat_of(strs):
    return np.frombuffer(b"".join(strs), np.uint8)


def string_values(strs, tag):
    """(wire bytes of each string's value, the values back to back): tag vi(len) bytes per string"""
    m = len(strs)
    if m == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.uint8)
    lens = lens_of(strs)
    return E._join([E._const_piece(m, bytes([tag])), varints(lens), (lens, flat_of(strs))])


def tiled_values(distinct, pattern, tag):
    """string_values of [distinct[p] for p in pattern] without building the list: each distinct value once, then gathered"""
    sz, flat = string_values(distinct, tag)
    start = np.concatenate([[0], np.cumsum(sz)])[:-1]
    pattern = np.asarray(pattern, np.int64)
    sizes = sz[pattern]
    if not len(pattern):
        return sizes, np.zeros(0, np.uint8)
    out_start = np.cumsum(sizes) - sizes
    idx = np.repeat(start[pattern] - out_start, sizes) + np.arange(int(sizes.sum()))
    return sizes, flat[idx]


def string_val_body(strs):
    return string_values(strs, 0x42)[1].tobytes()


def shape_bytes(dims):
    body = b"".join(b"\x12" + vi(len(d)) + d for d in ((b"\x08" + vi(x)) if x else b"" for x in dims))
    return b"\x12" + vi(len(body)) + body


def tensor_proto(body: bytes, dims) -> bytes:
    """a DT_STRING TensorProto whose string_val values are `body`"""
    return b"\x08\x07" + shape_bytes(dims) + body


def predict_request(name, version, inputs):
    """PredictRequest bytes of {key: TensorProto bytes}, entries in the deterministic runtime's order"""
    keys = [k.encode() if isinstance(k, str) else bytes(k) for k in inputs]
    vals = list(inputs.values())
    out = [E.model_spec(name, version)]
    for i in E.upb_order(keys):
        e = b"\x0a" + vi(len(keys[i])) + keys[i] + b"\x12" + vi(len(vals[i])) + vals[i]
        out.append(b"\x12" + vi(len(e)) + e)
    return b"".join(out)


def response_entry(key, tp: bytes) -> bytes:
    """one PredictResponse.outputs map entry"""
    kb = key.encode() if isinstance(key, str) else bytes(key)
    e = b"\x0a" + vi(len(kb)) + kb + b"\x12" + vi(len(tp)) + tp
    return b"\x0a" + vi(len(e)) + e


def concat_column(parts):
    """expected (data, offsets) of the concatenated decode: parts = each record's strings, in record order"""
    strs = [s for p in parts for s in p]
    off = np.zeros(len(strs) + 1, np.int64)
    np.cumsum(lens_of(strs), out=off[1:])
    return flat_of(strs), off


def padded_strings(parts, tail, pad):
    """the strings of the padded decode's column in position order: parts = (strings, dims) per record, tail = trailing dims"""
    out = []
    for strs, dims in parts:
        own = np.arange(int(np.prod(dims, dtype=np.int64))).reshape(dims) if len(strs) else None
        for row in range(dims[0]):
            for idx in np.ndindex(*tail):
                inside = all(i < d for i, d in zip(idx, dims[1:]))
                out.append(strs[int(own[(row,) + idx])] if inside else pad)
    return out


def padded_column(parts, tail, pad):
    """expected (data, offsets) of the padded decode"""
    return concat_column([padded_strings(parts, tail, pad)])


# ---- shared core: warp_copy_strings (+ the padded encode's CTA tier) ------------------------------------------------------
def tier(length, cta=False):
    """who copies a string: its lane, its warp, or (padded encode, cta=True) the whole CTA"""
    if length <= K_LANE:
        return "lane"
    return "cta" if cta and length > K_BLOCK else "warp"


def warp_rounds(lens, cta=False, active=None):
    """per warp-round of 32 consecutive strings: (lanes the warp copies one by one - the ballot's mask, tiers of the 32 lanes)"""
    lens = np.asarray(lens, np.int64)
    active = np.ones(len(lens), bool) if active is None else np.asarray(active)
    out = []
    for a in range(0, len(lens), WARP):
        t = [tier(int(x), cta) if ok else None for x, ok in zip(lens[a: a + WARP], active[a: a + WARP])]
        mask = sum(1 << i for i, x in enumerate(t) if x == "warp")
        out.append((mask, t))
    return out


def lane_mix(mask):
    """a name for a warp-round's ballot"""
    if mask == 0:
        return "all_lane"
    if mask == 0xFFFFFFFF:
        return "all_warp"
    if mask == 1:
        return "only_lane0"
    if mask == 1 << 31:
        return "only_lane31"
    if mask in (0x55555555, 0xAAAAAAAA):
        return "alternating"
    return "mixed"


def phases(addrs):
    return {int(a) & 15 for a in addrs}


# ---- padded encode ---------------------------------------------------------------------------------------------------------
class EncodeJob:
    """one (request, string input) job of the padded encode: its strings' lengths, in box order, and their column indexes"""

    def __init__(self, lens, index):
        self.lens = np.asarray(lens, np.int64)
        self.index = np.asarray(index, np.int64)
        ne = len(self.lens)
        self.tiles = max(-(-ne // K_VAR_THREADS), 1)                # an empty box takes a tile as well
        self.groups = -(-self.tiles // K_GROUP_TILES)
        t = np.arange(ne) // K_VAR_THREADS
        self.tile_of = t
        self.group_of_tile = np.arange(self.tiles) // K_GROUP_TILES
        self.cta_per_tile = np.bincount(t[self.lens > K_BLOCK], minlength=self.tiles)
        # a tile reads more than one run of the column when its strings' column indexes are not one stretch
        jump = np.r_[False, np.diff(self.index) != 1]
        self.crossing_tiles = set(t[jump & (np.r_[-1, t[:-1]] == t)].tolist())


def box_index(dims, r0, row):
    """column indexes of the box [r0 : r0 + row[0], :row[1], ...] of a column of shape dims, in C order"""
    bd = [int(row[0])] + [int(x) for x in row[1:]] if len(row) > 1 else [int(row[0])] + [int(d) for d in dims[1:]]
    return np.arange(int(np.prod(dims, dtype=np.int64))).reshape(dims)[(slice(r0, r0 + bd[0]),) + tuple(slice(0, x) for x in bd[1:])].ravel(), bd


# ---- concatenated decode ---------------------------------------------------------------------------------------------------
def concat_chunks(counts, ok):
    """counts / ok: [n_keys, n] per (key, record) pair, key-major as str_scan_kernel numbers them.  Returns (chunks per pair,
    chunk0 per pair, total chunks)"""
    counts, ok = np.asarray(counts, np.int64).ravel(), np.asarray(ok, bool).ravel()
    ch = np.where(ok, -(-counts // K_CHUNK), 0)
    c0 = np.cumsum(ch) - ch
    return ch, c0, int(ch.sum())


def pair_of(chunk0, c):
    """str_pair_of: the last pair whose first chunk is at or before c"""
    return int(np.searchsorted(chunk0, c, side="right")) - 1


def tied_pairs(ch, c0):
    """pairs that contribute no chunks and share their chunk0 with the pair that owns that chunk (the binary search's ties)"""
    return [q for q in range(len(ch)) if ch[q] == 0 and c0[q] < int(ch.sum()) and any(c0[p] == c0[q] and ch[p] for p in range(len(ch)))]


def concat_copy_grid(rec_lens, n_keys, sm_count):
    """CTAs of str_copy_kernel / str_fix_kernel, as b200tfs_decode_concat_strings sizes them (str_count_bound = rec_len / 2)"""
    bound = sum(n_keys * ((int(L) // 2) // K_CHUNK + 1) for L in rec_lens)
    per = K_STR_THREADS // 32
    return max(1, min(-(-bound // per), sm_count * 8))


def copy_strides(total_chunks, grid):
    """do the copy's warps take more than one chunk each?"""
    return total_chunks > grid * (K_STR_THREADS // 32)


def concat_scan(bytes_, ok, cap):
    """str_scan_kernel for one key: bytes_[r] and ok[r] (status OK before the scan) per record.  Returns (status per record:
    'ok' / 'size' / 'skip', first byte per record, offsets[m] or None).  A pair's bytes count in the running carry whether or not
    they fit, so every pair behind the first E_SIZE pair - zero-byte ones included - starts past data_cap and is E_SIZE too."""
    at, st, first, last = 0, [], [], None
    for b, o in zip(bytes_, ok):
        first.append(at)
        b = int(b) if o else 0
        if o and at + b > cap:
            st.append("size")
        elif o:
            st.append("ok")
            last = at + b
        else:
            st.append("skip")
        at += b
    return st, first, last


# ---- padded decode ---------------------------------------------------------------------------------------------------------
def padded_positions(keys):
    """keys: per key (parts = [(strings, dims)] per record, tail).  Returns per position, in the copy's global order:
    (key, record, own?, length)"""
    out = []
    for k, (parts, tail, pad) in enumerate(keys):
        for r, (strs, dims) in enumerate(parts):
            own = np.arange(int(np.prod(dims, dtype=np.int64))).reshape(dims)
            for row in range(dims[0]):
                for idx in np.ndindex(*tail):
                    inside = all(i < d for i, d in zip(idx, dims[1:]))
                    out.append((k, r, inside, len(strs[int(own[(row,) + idx])]) if inside else len(pad)))
    return out


def padded_rounds(pos):
    """the copy's warp-rounds (32 consecutive positions): how many span two records, and how many two keys"""
    rec = keys = 0
    for a in range(0, len(pos), WARP):
        w = pos[a: a + WARP]
        keys += len({p[0] for p in w}) > 1
        rec += len({(p[0], p[1]) for p in w}) > 1
    return rec, keys


def place_carries(dims):
    """PadStrPlace: own strings j > 0 whose last-axis index wraps to 0 (the full mixed radix runs again)"""
    m = int(np.prod(dims, dtype=np.int64))
    last = dims[-1] if len(dims) > 1 else m
    return sum(1 for j in range(1, m) if last and j % last == 0) if len(dims) > 1 else 0


# ---- index walk ------------------------------------------------------------------------------------------------------------
def string_fields(body_off, lens):
    """record offsets of every string value of a string_val body starting at body_off: (tag, first and last varint byte, first
    data byte)"""
    out, p = [], body_off
    for L in lens:
        n = len(vi(int(L)))
        out.append((p, p + 1, p + n, p + 1 + n))
        p += 1 + n + int(L)
    return out


def walk_lines(addr, fields):
    """the 128-byte lines (numbered from the record's base, addr rounded down) of every string's tag, length varint and first byte"""
    skew = int(addr) % LINE
    return [tuple((skew + x) // LINE for x in f) for f in fields]


def crossing_varints(lines):
    """strings whose tag and length varint do not lie in one line"""
    return [i for i, (t, v0, v1, _) in enumerate(lines) if len({t, v0, v1}) > 1]


def cold_jumps(addr, rec_len, fields):
    """reads of the walk (tags and varint bytes) that land on a line neither cached nor next to the one read before - a long
    string's skip - with the cursor's two-line cache opened on the record's first and last lines"""
    skew = int(addr) % LINE
    cache = [0, (skew + rec_len - 1) // LINE]
    victim, prev, jumps = 0, 0, 0
    for t, v0, v1, _ in fields:
        for x in range(t, v1 + 1):
            line = (skew + x) // LINE
            if line not in cache:
                jumps += line > prev + 1
                cache[victim] = line
                victim ^= 1
            prev = line
    return jumps


# ---- tf.Example bytes rows ----------------------------------------------------------------------------------------------------
def example_rounds(ne):
    """ex_write_bytes / ex_count_bytes: 32-string rounds of a row of ne strings, and the carries between them"""
    rounds = -(-int(ne) // WARP)
    return rounds, max(rounds - 1, 0)
