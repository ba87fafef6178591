"""A vectorised numpy reference for packed varints: the encoder and decoder of int_val, int64_val, uint32_val, uint64_val,
half_val and bool_val, and the geometry of the device kernels (csrc/varint_kernels.cuh) that the edge tests aim at.

tests/test_varint_reference_cpu.py pins this reference against the protobuf runtime and oracle/ref_port.py, and pins the
geometry constants below against the sources, so a retune cannot move the boundaries away from the tests.

Decoding follows the reference's order for one output: FromString refuses a malformed varint (E_PARSE), then
np.array(values, dtype) refuses a value out of the dtype's range (E_RANGE), then reshape() refuses the element count (E_SHAPE).
"""
import numpy as np

import golden_util as G

# ---- the kernels' geometry (plan.h, kernels.cu, codec_host.cpp) ---------------------------------------------------------
ENC_TILE = 2048            # kVarTileElems: elements per encode tile
GROUP_TILES = 256          # kVarGroupTiles: tiles per counter group
DEC_TILE = 8192            # kVarTileBytes: wire bytes per decode tile (an aligned window)
TINY = 32                  # kTinyVarElems: inputs this small are framed by the framing kernel itself
HOST_MEASURE = 4096        # host_measurable_varint: host inputs up to this many elements are measured on the host
ENC_GROUP_ELEMS = ENC_TILE * GROUP_TILES      # 524 288 elements: the first encode group boundary
DEC_GROUP_BYTES = DEC_TILE * GROUP_TILES      # 2 MiB of wire: the first decode group boundary

# ---- status codes (include/b200tfs.h) ----------------------------------------------------------------------------------
OK, E_SHAPE, E_PARSE, E_RANGE = 0, -2, -4, -9
EXCEPTION = {OK: None, E_SHAPE: "ValueError", E_PARSE: "DecodeError", E_RANGE: "OverflowError"}

# DataType enum -> (TensorProto value field, numpy dtype of the tensor, field holds int32 values)
DTYPES = {
    3: (7, np.int32, True), 4: (7, np.uint8, True), 5: (7, np.int16, True), 6: (7, np.int8, True), 17: (7, np.uint16, True),
    9: (10, np.int64, False), 22: (16, np.uint32, False), 23: (17, np.uint64, False), 10: (11, np.bool_, False),
    19: (13, np.float16, True),
}
NAMES = {3: "int32", 4: "uint8", 5: "int16", 6: "int8", 17: "uint16", 9: "int64", 22: "uint32", 23: "uint64", 10: "bool", 19: "half"}
RANGE = {4: (0, 255), 5: (-32768, 32767), 6: (-128, 127), 17: (0, 65535)}


def wire_words(values, dtype):
    """The 64-bit words the protobuf runtime writes for a tensor's elements: signed types sign-extended, half as its bits."""
    a = np.ascontiguousarray(values).reshape(-1)
    if dtype == 19:
        return a.view(np.uint16).astype(np.uint64)
    if dtype == 10:
        return a.astype(np.uint64)
    if np.issubdtype(a.dtype, np.signedinteger):
        return a.astype(np.int64).view(np.uint64)
    return a.astype(np.uint64)


def varint_lengths(words):
    """Bytes of each varint: ceil(bit length / 7), at least one."""
    w = np.asarray(words, dtype=np.uint64)
    n = np.ones(w.shape, dtype=np.int64)
    for k in range(1, 10):
        n += (w >= np.uint64(1 << (7 * k))).astype(np.int64)
    return n


def encode_words(words):
    """The packed varints of 64-bit words, as bytes."""
    w = np.asarray(words, dtype=np.uint64).reshape(-1)
    if not w.size:
        return b""
    lens = varint_lengths(w)
    k = np.arange(10, dtype=np.uint64)
    groups = ((w[:, None] >> (np.uint64(7) * k)) & np.uint64(0x7F)).astype(np.uint8)
    groups |= np.where(k[None, :] < (lens[:, None] - 1).astype(np.uint64), np.uint8(0x80), np.uint8(0))
    return groups[np.arange(10)[None, :] < lens[:, None]].tobytes()


def encode(values, dtype):
    return encode_words(wire_words(values, dtype))


def packed_len(values, dtype):
    return int(varint_lengths(wire_words(values, dtype)).sum())


def field(dtype, chunks):
    """The packed occurrences of a dtype's value field (uint32_val and uint64_val have two-byte tags)."""
    tag = G.vi((DTYPES[dtype][0] << 3) | 2)
    return b"".join(tag + G.vi(len(c)) + bytes(c) for c in chunks)


def tensor_proto(values, dtype, dims=None):
    """TensorProto(dtype, tensor_shape, <value field>=values).SerializeToString()."""
    dims = list(np.shape(values)) if dims is None else list(dims)
    return tensor_header(dtype, dims, packed_len(values, dtype)) + encode(values, dtype)


def tensor_header(dtype, dims, length):
    """The framing in front of a packed payload of `length` bytes (everything of tensor_proto but the payload)."""
    if not length:
        return G.tproto(dtype, dims, b"")
    return G.tproto(dtype, dims, G.vi((DTYPES[dtype][0] << 3) | 2) + G.vi(length))


def split_varints(wire):
    """(start, length) of every varint of a packed run, and whether the last one is unterminated."""
    b = np.frombuffer(bytes(wire), dtype=np.uint8)
    ends = np.flatnonzero(b < 0x80)
    starts = np.concatenate([[0], ends[:-1] + 1]).astype(np.int64) if ends.size else np.zeros(0, np.int64)
    return starts, (ends - starts + 1).astype(np.int64), bool(b.size and b[-1] >= 0x80)


def decode_words(wire):
    """(64-bit words, malformed): every varint of a packed run; a varint longer than ten bytes or an unterminated last one
    makes the run malformed (the words of the first ten bytes are still returned)."""
    b = np.frombuffer(bytes(wire), dtype=np.uint8)
    starts, lens, open_end = split_varints(wire)
    if not starts.size:
        return np.zeros(0, np.uint64), open_end
    total = int(lens.sum())         # bytes up to the last terminator
    pos = np.arange(total, dtype=np.int64) - np.repeat(starts, lens)
    keep = pos < 10
    contrib = (b[:total][keep].astype(np.uint64) & np.uint64(0x7F)) << (np.uint64(7) * pos[keep].astype(np.uint64))
    owner = np.repeat(np.arange(starts.size), lens)[keep]
    words = np.zeros(starts.size, dtype=np.uint64)
    np.bitwise_or.at(words, owner, contrib)
    return words, bool(open_end or (lens > 10).any())


def values_of(words, dtype):
    """The elements a TensorProto field of 64-bit words reads back as: int_val and half_val truncated to 32 bits, uint32_val to
    32 bits, bool_val nonzero; None for an int_val value outside an 8- or 16-bit dtype's range."""
    w = np.asarray(words, dtype=np.uint64)
    field, np_type, int32_field = DTYPES[dtype]
    if dtype == 10:
        return w != 0
    if dtype == 19:
        return (w & np.uint64(0xFFFF)).astype(np.uint16).view(np.float16)
    if int32_field:
        x = (w & np.uint64(0xFFFFFFFF)).astype(np.uint32).view(np.int32).astype(np.int64)
        if dtype in RANGE:
            lo, hi = RANGE[dtype]
            if ((x < lo) | (x > hi)).any():
                return None
        return x.astype(np_type)
    if dtype == 22:
        return (w & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    return w.view(np.int64) if dtype == 9 else w


def decode(chunks, dtype, n_elems, tolerant=False):
    """(values, status) of one output whose packed occurrences are `chunks` and whose shape holds n_elems elements.
    tolerant: TensorFlow's MakeNdarray padding - fewer values than elements repeat the last one, none give zeros."""
    if isinstance(chunks, (bytes, bytearray)):
        chunks = [chunks]
    parts, bad = [], False
    for c in chunks:
        words, malformed = decode_words(c)
        parts.append(words)
        bad = bad or malformed
    if bad:
        return None, E_PARSE
    words = np.concatenate(parts) if parts else np.zeros(0, np.uint64)
    vals = values_of(words, dtype)
    if vals is None:
        return None, E_RANGE
    n = vals.size
    if n == n_elems:
        return vals, OK
    if tolerant and n < n_elems:
        out = np.zeros(n_elems, dtype=vals.dtype)
        if n:
            out[:n] = vals
            out[n:] = vals[-1]
        return out, OK
    return None, E_SHAPE
