// walker.h - the PredictResponse / TensorProto tag walk that the decode kernels run (one lane per
// record).  It tabulates where every output's values lie in the wire so the unpack code can move
// them; it moves no payload bytes itself.
//
// Behaviour follows what the reference observes through PredictResponse.FromString
// (prediction_service_pb2_grpc.py:53 -> protobuf runtime) + extract_shape / tensor_proto_to_ndarray
// (tensors.py:38-46), case by case as pinned in tests/golden/decode.json (SURVEY 8a D1-D5):
//   fields in any order; scalar dtype: last wins; tensor_shape repeated: dims concatenate; packed
//   fields split over several occurrences and unpacked elements: concatenate in wire order; unknown
//   fields (varint / fixed / length-delimited / groups) skipped; duplicate map key: last entry wins;
//   truncated input, tag 0, bad UTF-8 in a string field, packed fixed32 length % 4 != 0: parse error.
//
// Shape of the code: ONE cursor per record (32-bit offsets relative to the record start, nested
// messages narrow `end` and restore it), no recursion, every helper force-inlined, so on the device
// the whole walk state lives in registers and the only memory touched is the two-line cache below
// and the output table.  The same source compiles for the host, where tests/native replays the golden
// vectors through it.
#pragma once
#include "../../include/b200tfs.h"
#include "wire.h"

namespace b200tfs {

// One lane chasing bytes through HBM pays a DRAM round trip per miss, so it reads the wire through
// a cache of two 128-byte lines (shared memory), each filled with eight independent 16-byte loads.
// The canonical response (header ... payload ... model_spec) costs two misses, both issued up front.
struct Cursor {
  const uint8_t* rec;  // first byte of the record
  uint32_t p;          // offset of the next unread byte, relative to rec
  uint32_t end;        // limit of the message being walked
  int32_t err;         // sticky B200TFS_E_PARSE
  // device only: the line cache
  const uint8_t* base; // rec rounded down to 128
  uint8_t* buf;        // 256 bytes of shared memory
  uint32_t skew;       // rec - base
  uint32_t line0, line1, victim;  // cached line numbers (relative to base), ~0 = empty
};

#if defined(__CUDACC__)
// out of line: a miss is rare (two per canonical response) and its sixteen vector accesses, inlined at every one of the walk's
// ~100 byte reads, were most of the walk's 230 KB of SASS
__device__ __noinline__ void cur_fill(Cursor& c, uint32_t slot, uint32_t line) {
  const uint4* g = reinterpret_cast<const uint4*>(c.base + ((uint64_t)line << 7));
  uint4 t0 = g[0], t1 = g[1], t2 = g[2], t3 = g[3], t4 = g[4], t5 = g[5], t6 = g[6], t7 = g[7];
  uint4* s = reinterpret_cast<uint4*>(c.buf + 128 * slot);
  s[0] = t0; s[1] = t1; s[2] = t2; s[3] = t3; s[4] = t4; s[5] = t5; s[6] = t6; s[7] = t7;
}
// bind a cursor to a record and fetch its first and last line together
__device__ __forceinline__ void cur_open(Cursor& c, const uint8_t* rec, uint32_t len, uint8_t* smem256) {
  c.rec = rec; c.p = 0; c.end = len; c.err = 0;
  c.base = reinterpret_cast<const uint8_t*>((uintptr_t)rec & ~(uintptr_t)127);
  c.skew = (uint32_t)(rec - c.base);
  c.buf = smem256; c.victim = 0; c.line0 = c.line1 = ~0u;
  if (len) {
    const uint32_t lb = (c.skew + len - 1) >> 7;
    const uint4* ga = reinterpret_cast<const uint4*>(c.base);
    const uint4* gb = reinterpret_cast<const uint4*>(c.base + ((uint64_t)lb << 7));
    uint4 x0 = ga[0], x1 = ga[1], x2 = ga[2], x3 = ga[3], x4 = ga[4], x5 = ga[5], x6 = ga[6], x7 = ga[7];
    uint4 y0 = gb[0], y1 = gb[1], y2 = gb[2], y3 = gb[3], y4 = gb[4], y5 = gb[5], y6 = gb[6], y7 = gb[7];
    uint4* s = reinterpret_cast<uint4*>(c.buf);
    s[0] = x0; s[1] = x1; s[2] = x2; s[3] = x3; s[4] = x4; s[5] = x5; s[6] = x6; s[7] = x7;
    s[8] = y0; s[9] = y1; s[10] = y2; s[11] = y3; s[12] = y4; s[13] = y5; s[14] = y6; s[15] = y7;
    c.line0 = 0; c.line1 = lb;
  }
}
#endif
inline void cur_open_host(Cursor& c, const uint8_t* rec, uint32_t len) {
  c.rec = rec; c.p = 0; c.end = len; c.err = 0;
  c.base = rec; c.buf = nullptr; c.skew = 0; c.line0 = c.line1 = ~0u; c.victim = 0;
}

// byte at record offset q
B2_HD uint8_t rd8(Cursor& c, uint32_t q) {
#if defined(__CUDA_ARCH__)
  const uint32_t a = q + c.skew, line = a >> 7;
  if (line == c.line0) return c.buf[a & 127];
  if (line == c.line1) return c.buf[128 + (a & 127)];
  const uint32_t k = c.victim;
  c.victim = k ^ 1;
  cur_fill(c, k, line);
  if (k) c.line1 = line; else c.line0 = line;
  return c.buf[128 * k + (a & 127)];
#else
  return c.rec[q];
#endif
}

B2_HD uint64_t rd_varint(Cursor& c) {
  uint64_t v = 0;
#pragma unroll 1
  for (int i = 0; i < 10; ++i) {
    if (c.p >= c.end) { c.err = B200TFS_E_PARSE; return 0; }
    const uint8_t b = rd8(c, c.p++);
    v |= (uint64_t)(b & 0x7F) << (7 * i);  // bits past 64 fall off, as in the runtime
    if (!(b & 0x80)) return v;
  }
  c.err = B200TFS_E_PARSE;  // 10 continuation bytes
  return 0;
}

// tag: at most 5 bytes (the runtime refuses a longer one, even of a small value), must fit 32 bits, field number != 0
B2_HD uint32_t rd_tag(Cursor& c) {
  uint64_t t = 0;
#pragma unroll 1
  for (int i = 0; i < 5; ++i) {
    if (c.p >= c.end) break;
    const uint8_t b = rd8(c, c.p++);
    t |= (uint64_t)(b & 0x7F) << (7 * i);
    if (!(b & 0x80)) {
      if (t > 0xFFFFFFFFull || (t >> 3) == 0) break;
      return (uint32_t)t;
    }
  }
  c.err = B200TFS_E_PARSE;   // truncated, a sixth byte, past 32 bits, or field 0
  return 0;
}

// length prefix: bounded by the enclosing message (and by int32, like the runtime)
B2_HD uint32_t rd_len(Cursor& c) {
  const uint64_t n = rd_varint(c);
  if (c.err) return 0;
  if (n > 0x7FFFFFFFull || n > (uint64_t)(c.end - c.p)) { c.err = B200TFS_E_PARSE; return 0; }
  return (uint32_t)n;
}

// Skip one non-group field body (tag already consumed).
B2_HD void skip_scalar(Cursor& c, uint32_t wt) {
  if (wt == WT_VARINT) { (void)rd_varint(c); return; }
  if (wt == WT_I64) { if (c.end - c.p < 8) c.err = B200TFS_E_PARSE; else c.p += 8; return; }
  if (wt == WT_I32) { if (c.end - c.p < 4) c.err = B200TFS_E_PARSE; else c.p += 4; return; }
  if (wt == WT_LEN) { const uint32_t n = rd_len(c); if (!c.err) c.p += n; return; }
  c.err = B200TFS_E_PARSE;  // stray END_GROUP, wire types 6 and 7
}

// Skip one field body of any wire type.  Groups nest: the open field numbers are kept on a small
// explicit stack (depth <= 16; deeper is treated as malformed); an END_GROUP that does not close
// the innermost open group is malformed.
B2_HD void skip_field(Cursor& c, uint32_t tag) {
  const uint32_t wt = tag & 7;
  if (wt != WT_SGROUP) { skip_scalar(c, wt); return; }
  uint32_t open[16];
  int depth = 0;
  open[depth++] = tag >> 3;
#pragma unroll 1
  while (depth > 0 && !c.err) {
    if (c.p >= c.end) { c.err = B200TFS_E_PARSE; return; }
    const uint32_t t = rd_tag(c);
    if (c.err) return;
    const uint32_t w2 = t & 7;
    if (w2 == WT_SGROUP) {
      if (depth >= 16) { c.err = B200TFS_E_PARSE; return; }
      open[depth++] = t >> 3;
    } else if (w2 == WT_EGROUP) {
      if (open[depth - 1] != (t >> 3)) { c.err = B200TFS_E_PARSE; return; }
      --depth;
    } else {
      skip_scalar(c, w2);
    }
  }
}

// Structural UTF-8 check the runtime applies to proto3 `string` fields (shortest form, no
// surrogates, <= U+10FFFF) over record bytes [off, off+n).
B2_HD bool utf8_ok(Cursor& c, uint32_t off, uint32_t n) {
  uint32_t i = 0;
#pragma unroll 1
  while (i < n) {
    const uint8_t b = rd8(c, off + i);
    if (b < 0x80) { ++i; continue; }
    uint32_t need, cp;
    if (b >= 0xC2 && b <= 0xDF) { need = 1; cp = b & 0x1F; }
    else if (b >= 0xE0 && b <= 0xEF) { need = 2; cp = b & 0x0F; }
    else if (b >= 0xF0 && b <= 0xF4) { need = 3; cp = b & 0x07; }
    else return false;
    if (n - i - 1 < need) return false;
    for (uint32_t k = 1; k <= need; ++k) {
      const uint8_t x = rd8(c, off + i + k);
      if ((x & 0xC0) != 0x80) return false;
      cp = (cp << 6) | (x & 0x3F);
    }
    if (need == 2 && (cp < 0x800 || (cp >= 0xD800 && cp <= 0xDFFF))) return false;
    if (need == 3 && (cp < 0x10000 || cp > 0x10FFFF)) return false;
    i += need + 1;
  }
  return true;
}

// a length-delimited string field: validate, return its record offset, step over it
B2_HD uint32_t rd_string(Cursor& c, uint32_t* len) {
  const uint32_t n = rd_len(c);
  if (c.err) { *len = 0; return 0; }
  const uint32_t at = c.p;
  if (!utf8_ok(c, at, n)) { c.err = B200TFS_E_PARSE; *len = 0; return 0; }
  c.p += n;
  *len = n;
  return at;
}

// Structural validation of the message-typed TensorProto fields this path never reads
// (resource_handle_val = 14, variant_val = 15).  The runtime parses them recursively, so malformed
// bytes inside them fail the whole response; this walks the same schemas (resource_handle.proto:16-42,
// tensor.proto:87-94, tensor_shape.proto:13-46) with an explicit stack instead of recursion
// (variant_val can nest TensorProtos): tags, lengths, packed-field shape and UTF-8 of string fields.
enum NestedType : uint32_t { NT_TENSOR = 0, NT_SHAPE, NT_DIM, NT_RESOURCE, NT_DTYPE_AND_SHAPE, NT_VARIANT };

// what field `f` of message type `t` is: 0 = unknown/scalar (skip by wire type), 1 = string (UTF-8),
// 2 = packed-or-scalar numeric (TensorProto value fields), 0x10 | type = sub-message to descend into
B2_HD uint32_t nested_field_kind(uint32_t t, uint32_t f) {
  switch (t) {
    case NT_TENSOR:
      if (f == F_SHAPE) return 0x10 | NT_SHAPE;
      if (f == F_RESOURCE) return 0x10 | NT_RESOURCE;
      if (f == F_VARIANT) return 0x10 | NT_VARIANT;
      if (scalar_wire_type(f) != 0xFFu) return 2;
      return 0;
    case NT_SHAPE: return f == 2 ? (0x10 | NT_DIM) : 0;
    case NT_DIM: return f == 2 ? 1 : 0;
    case NT_RESOURCE:
      if (f == 1 || f == 2 || f == 3 || f == 5) return 1;
      return f == 6 ? (0x10 | NT_DTYPE_AND_SHAPE) : 0;
    case NT_DTYPE_AND_SHAPE: return f == 2 ? (0x10 | NT_SHAPE) : 0;
    default:  // NT_VARIANT
      if (f == 1) return 1;
      return f == 3 ? (0x10 | NT_TENSOR) : 0;
  }
}

constexpr int kNestedDepth = 16;

// validate a sub-message of `type` occupying [c.p, c.p + len); leaves c.p at its end.  Returns false
// (without flagging a parse error) only when nesting exceeds kNestedDepth.
B2_HD bool validate_nested(Cursor& c, uint32_t type, uint32_t len) {
  uint32_t end_stack[kNestedDepth];
  uint8_t type_stack[kNestedDepth];
  int depth = 0;
  const uint32_t outer = c.end;
  c.end = c.p + len;
#pragma unroll 1
  for (;;) {
    if (c.err) break;
    if (c.p >= c.end) {  // this message is complete: back to its parent
      if (depth == 0) break;
      --depth;
      c.end = end_stack[depth]; type = type_stack[depth];
      continue;
    }
    const uint32_t tag = rd_tag(c);
    if (c.err) break;
    const uint32_t f = tag >> 3, wt = tag & 7;
    const uint32_t kind = nested_field_kind(type, f);
    if (kind == 1 && wt == WT_LEN) { uint32_t k; (void)rd_string(c, &k); }
    else if (kind == 2 && wt == WT_LEN) {
      const uint32_t n = rd_len(c);
      if (c.err) break;
      const uint32_t fw = fixed_wire_width(f);
      if (fw ? (n % fw) != 0 : (n && (rd8(c, c.p + n - 1) & 0x80))) { c.err = B200TFS_E_PARSE; break; }
      c.p += n;
    } else if ((kind & 0x10) && wt == WT_LEN) {
      const uint32_t n = rd_len(c);
      if (c.err) break;
      if (depth >= kNestedDepth) { c.end = outer; return false; }
      end_stack[depth] = c.end; type_stack[depth] = (uint8_t)type;
      ++depth;
      c.end = c.p + n; type = kind & 0xF;
    } else skip_field(c, tag);
  }
  c.end = outer;
  return true;
}

// Begin a fresh output record: only the fields the walk accumulates into.
B2_HD void out_begin(b200tfs_output& o) {
  o.key_off = 0; o.key_len = 0; o.dtype = 0; o.rank = 0; o.flags = 0; o.value_field = 0; o.n_runs = 0;
  o.content_off = 0; o.content_len = 0; o.msg_off = 0; o.msg_len = 0;
  o.n_elems = 0; o.dst_bytes = 0; o.n_strings = 0; o.dst_off = 0; o.status = B200TFS_OK;
  o.n_inline = 0; o.spill_rec = 0; o.spill_seq = 0;
}

// What does not fit the table's inline arrays - dims past B200TFS_MAX_RANK, value runs past B200TFS_MAX_RUNS - is
// appended to the record's spill region (global memory on the device; the two-phase parse sizes it and runs again
// when a record wants more: `used` keeps counting past `cap`).  Entries carry the ordinal of the map entry they
// belong to, so that a later entry with the same key (which replaces the earlier one) is told apart.
struct SpillEntry {
  uint32_t kind;        // 1 = dim (run.off holds the size), 2 = value run
  uint32_t seq;         // map-entry ordinal inside the record
  b200tfs_run run;
};
struct SpillArea {
  SpillEntry* e;        // this record's region (nullptr when cap == 0)
  uint32_t cap, used;
};
enum : uint32_t { SPILL_DIM = 1, SPILL_RUN = 2 };

// Walk state of one map entry that does not belong in the table.
struct WalkAux {
  uint32_t seq;         // ordinal of the entry being walked
  uint32_t last_spill;  // index (in the record's region) of the last spilled RUN of this entry, ~0u = none
  bool too_deep;        // variant_val nesting beyond kNestedDepth
};
B2_HD void aux_begin(WalkAux& a, uint32_t seq) { a.seq = seq; a.last_spill = ~0u; a.too_deep = false; }

B2_HD void spill_push(SpillArea& sp, uint32_t kind, uint32_t seq, const b200tfs_run& r) {
  if (sp.used < sp.cap) { SpillEntry& e = sp.e[sp.used]; e.kind = kind; e.seq = seq; e.run = r; }
  ++sp.used;
}

B2_HD void add_dim(b200tfs_output& o, SpillArea& sp, const WalkAux& a, int64_t size) {
  if (o.rank < B200TFS_MAX_RANK) o.dims[o.rank] = size;
  else {
    b200tfs_run r; r.off = (uint64_t)size; r.len = 0; r.count = 0; r.stride = 0; r.field = 0;
    spill_push(sp, SPILL_DIM, a.seq, r);
    o.flags |= B200TFS_OF_SPILLED;
  }
  ++o.rank;
}

// One more piece of values: `len` bytes at record offset `off`, from TensorProto field `field`.  Short pieces
// (unpacked scalar elements: at most ten bytes) that follow the previous one at a constant distance extend its run,
// so that a field written element by element - however long - stays ONE table entry; longer pieces (packed
// occurrences) each get a run of their own and keep the tiled copy path.
constexpr uint32_t kCoalesceMax = 16;
B2_HD void add_piece(b200tfs_output& o, SpillArea& sp, WalkAux& a, uint32_t field, uint32_t off, uint32_t len) {
  b200tfs_run* last = nullptr;
  if (o.n_runs > 0) {
    if (o.n_runs <= B200TFS_MAX_RUNS) last = &o.runs[o.n_runs - 1];
    else if (a.last_spill < sp.cap) last = &sp.e[a.last_spill].run;
  }
  if (last && len <= kCoalesceMax && last->field == field && last->len == len) {
    if (last->count == 1) {
      if (off > last->off && off - last->off >= len) { last->stride = (uint32_t)(off - last->off); last->count = 2; return; }
    } else if (off == last->off + (uint64_t)last->count * last->stride && last->count < 0xFFFFFFFFu) { ++last->count; return; }
  }
  b200tfs_run r; r.off = off; r.len = len; r.count = 1; r.stride = 0; r.field = field;
  if (o.n_runs < B200TFS_MAX_RUNS) o.runs[o.n_runs] = r;
  else {
    a.last_spill = sp.used;
    spill_push(sp, SPILL_RUN, a.seq, r);
    o.flags |= B200TFS_OF_SPILLED;
  }
  ++o.n_runs;
}

// TensorShapeProto (tensor_shape.proto:13-46) in [c.p, c.end): dims append (merge); Dim.size last
// wins inside a Dim; Dim.name validated and ignored (tensors.py:38-39).
B2_HD void walk_shape(Cursor& c, b200tfs_output& o, SpillArea& sp, WalkAux& a) {
#pragma unroll 1
  while (c.p < c.end && !c.err) {
    const uint32_t tag = rd_tag(c);
    if (c.err) return;
    if (tag != tag_of(2, WT_LEN)) { skip_field(c, tag); continue; }  // unknown_rank (3) and anything else
    const uint32_t n = rd_len(c);
    if (c.err) return;
    const uint32_t outer = c.end;
    c.end = c.p + n;
    int64_t size = 0;
#pragma unroll 1
    while (c.p < c.end && !c.err) {
      const uint32_t t = rd_tag(c);
      if (c.err) break;
      if (t == tag_of(1, WT_VARINT)) size = (int64_t)rd_varint(c);
      else if (t == tag_of(2, WT_LEN)) { uint32_t k; (void)rd_string(c, &k); }
      else skip_field(c, t);
    }
    c.end = outer;
    if (c.err) return;
    add_dim(o, sp, a, size);
  }
}

// One TensorProto (tensor.proto:14-84) in [c.p, c.end); accumulates into o so a repeated `value` merges.
// Every offset written to the table is relative to the record start.
B2_HD void walk_tensor(Cursor& c, b200tfs_output& o, SpillArea& sp, WalkAux& a) {
#pragma unroll 1
  while (c.p < c.end && !c.err) {
    const uint32_t tag = rd_tag(c);
    if (c.err) return;
    const uint32_t field = tag >> 3, wt = tag & 7;
    if (field == F_DTYPE && wt == WT_VARINT) {
      o.dtype = (int32_t)(uint32_t)rd_varint(c);
    } else if (field == F_SHAPE && wt == WT_LEN) {
      const uint32_t n = rd_len(c);
      if (c.err) return;
      const uint32_t outer = c.end;
      c.end = c.p + n;
      walk_shape(c, o, sp, a);
      c.end = outer;
    } else if (field == F_CONTENT && wt == WT_LEN) {
      const uint32_t n = rd_len(c);
      if (c.err) return;
      o.content_off = c.p; o.content_len = n;  // `bytes`: last occurrence replaces
      c.p += n;
    } else if (field == F_STRING && wt == WT_LEN) {
      const uint32_t n = rd_len(c);
      if (c.err) return;
      o.n_strings += 1;
      c.p += n;
    } else if (scalar_wire_type(field) != 0xFFu && (wt == WT_LEN || wt == scalar_wire_type(field))) {
      uint32_t off, len;
      if (wt == WT_LEN) {
        len = rd_len(c);
        if (c.err) return;
        off = c.p;
        const uint32_t fw = fixed_wire_width(field);
        if (fw) {
          if (len % fw) { c.err = B200TFS_E_PARSE; return; }  // packed fixed32/64 must be whole elements
        } else if (len && (rd8(c, off + len - 1) & 0x80)) {
          c.err = B200TFS_E_PARSE; return;                    // packed varints must end on a terminator
        }
        c.p += len;
      } else {
        off = c.p;
        skip_scalar(c, wt);
        if (c.err) return;
        len = c.p - off;
        o.flags |= B200TFS_OF_UNPACKED;
      }
      if (len) add_piece(o, sp, a, field, off, len);
    } else if ((field == F_RESOURCE || field == F_VARIANT) && wt == WT_LEN) {
      const uint32_t n = rd_len(c);
      if (c.err) return;
      if (!validate_nested(c, field == F_RESOURCE ? NT_RESOURCE : NT_VARIANT, n)) a.too_deep = true;  // too deep: NONCANONICAL
    } else {
      if (field > 17) o.flags |= B200TFS_OF_HAS_UNKNOWN;
      skip_field(c, tag);  // version_number, mismatched wire types, unknown
    }
  }
}

// the k-th spilled entry of `kind` that belongs to map entry `seq` (nullptr if absent / beyond the region)
B2_HD SpillEntry* spill_find(SpillArea& sp, uint32_t kind, uint32_t seq, uint32_t k) {
  const uint32_t n = sp.used < sp.cap ? sp.used : sp.cap;
  for (uint32_t i = 0; i < n; ++i)
    if (sp.e[i].kind == kind && sp.e[i].seq == seq) { if (k == 0) return &sp.e[i]; --k; }
  return nullptr;
}

// Every varint of `count` pieces of `len` bytes, `stride` apart, ends within ten bytes (the walk has checked that each piece
// ends on a terminator).
B2_HD bool varint_pieces_ok(Cursor& c, const b200tfs_run& r) {
#pragma unroll 1
  for (uint32_t q = 0; q < r.count; ++q) {
    uint32_t run = 0;
#pragma unroll 1
    for (uint32_t i = 0; i < r.len; ++i) {
      run = (rd8(c, (uint32_t)r.off + q * r.stride + i) & 0x80) ? run + 1 : 0;
      if (run >= 10) return false;
    }
  }
  return true;
}

// Packed varints of a field the dtype does not select are dropped from the table, so no varint decode kernel ever reads them;
// the runtime parses them all the same and refuses the whole message when one is malformed.  Check those here (they are
// absent from the responses a server writes, so this costs nothing there).
B2_HD bool foreign_varints_ok(Cursor& c, const b200tfs_output& o, const SpillArea& sp, const WalkAux& a, uint32_t field) {
  const int inl = o.n_runs < B200TFS_MAX_RUNS ? o.n_runs : B200TFS_MAX_RUNS;
  for (int i = 0; i < inl; ++i)
    if (o.runs[i].field != field && !fixed_wire_width(o.runs[i].field) && !varint_pieces_ok(c, o.runs[i])) return false;
  const uint32_t n = sp.used < sp.cap ? sp.used : sp.cap;
  for (uint32_t i = 0; i < n && o.n_runs > B200TFS_MAX_RUNS; ++i) {
    const SpillEntry& e = sp.e[i];
    if (e.kind == SPILL_RUN && e.seq == a.seq && e.run.field != field && !fixed_wire_width(e.run.field) && !varint_pieces_ok(c, e.run))
      return false;
  }
  return true;
}

// Settle dtype -> field, keep that field's runs, element counts.  Mirrors what
// tensor_proto_to_ndarray (tensors.py:42-46) would conclude from the parsed message.
B2_HD void finalize_output(Cursor& c, b200tfs_output& o, SpillArea& sp, const WalkAux& a) {
  o.spill_seq = a.seq;
  if (!foreign_varints_ok(c, o, sp, a, dtype_info(o.dtype).field)) { c.err = B200TFS_E_PARSE; return; }
  if (a.too_deep) { o.status = B200TFS_E_NONCANONICAL; o.n_runs = 0; o.n_inline = 0; return; }
  const DtypeInfo di = dtype_info(o.dtype);
  if (di.field == 0) { o.status = B200TFS_E_KEY; o.n_runs = 0; o.n_inline = 0; return; }  // types.py:40 KeyError
  o.value_field = (int32_t)di.field;
  uint64_t total = 0;
  bool gathered = false;
  int kept = 0;
  const int inl = o.n_runs < B200TFS_MAX_RUNS ? o.n_runs : B200TFS_MAX_RUNS;
  for (int i = 0; i < inl; ++i) {
    if (o.runs[i].field == di.field) {
      o.runs[kept] = o.runs[i];
      total += (uint64_t)o.runs[i].len * o.runs[i].count;
      gathered = gathered || o.runs[i].count > 1;
      ++kept;
    }
  }
  o.n_inline = (uint32_t)kept;
  if (o.n_runs > B200TFS_MAX_RUNS) {   // spilled runs stay where they are (the host keeps those of this field)
    const uint32_t n = sp.used < sp.cap ? sp.used : sp.cap;
    for (uint32_t i = 0; i < n; ++i) {
      const SpillEntry& e = sp.e[i];
      if (e.kind == SPILL_RUN && e.seq == a.seq && e.run.field == di.field) {
        total += (uint64_t)e.run.len * e.run.count;
        gathered = gathered || e.run.count > 1;
        ++kept;
      }
    }
  }
  o.n_runs = kept;
  if (kept > 1 || gathered) o.flags |= B200TFS_OF_MULTI_CHUNK;
  if (o.content_len) o.flags |= B200TFS_OF_TENSOR_CONTENT;
  if (o.rank == 0) o.flags |= B200TFS_OF_RANK0;
  // prod(dims) with at most one -1
  uint64_t prod = 1; int infer = -1; bool bad = false;
  for (int i = 0; i < o.rank; ++i) {
    int64_t d;
    if (i < B200TFS_MAX_RANK) d = o.dims[i];
    else { const SpillEntry* e = spill_find(sp, SPILL_DIM, a.seq, (uint32_t)(i - B200TFS_MAX_RANK)); d = e ? (int64_t)e->run.off : 1; }
    if (d == -1 && infer < 0) { infer = i; continue; }
    if (d < 0) { bad = true; break; }
    if (d != 0 && prod > 0xFFFFFFFFFFFFFFFFull / (uint64_t)d) { bad = true; break; }
    prod *= (uint64_t)d;
  }
  if (bad) { o.status = B200TFS_E_SHAPE; return; }
  auto set_dim = [&](int i, int64_t v) {
    if (i < B200TFS_MAX_RANK) o.dims[i] = v;
    else { SpillEntry* e = spill_find(sp, SPILL_DIM, a.seq, (uint32_t)(i - B200TFS_MAX_RANK)); if (e) e->run.off = (uint64_t)v; }
  };
  // n_elems / dst_bytes describe the SHAPE (once it is fully known), also when the values do not match it:
  // the tolerant decoder needs them to accept tensor_content in place of the typed field
  if (di.kind == VK_FIXED) {
    const uint64_t count = total / di.elem_size;  // complex: interleaved (re, im) pairs, TF convention
    if (total % di.elem_size) { o.status = B200TFS_E_SHAPE; return; }
    if (infer >= 0) {
      if (prod == 0 || count % prod) { o.status = B200TFS_E_SHAPE; return; }
      set_dim(infer, (int64_t)(count / prod)); prod = count; o.flags |= B200TFS_OF_DIM_INFERRED;
    }
    o.n_elems = prod; o.dst_bytes = prod * di.elem_size;
    if (count != prod) { o.status = B200TFS_E_SHAPE; return; }  // reshape() ValueError: no broadcast, no padding
  } else if (di.kind == VK_VARINT || di.kind == VK_BOOL) {
    o.flags |= B200TFS_OF_VARINT;
    if (infer >= 0) { o.status = B200TFS_E_NONCANONICAL; return; }
    o.n_elems = prod; o.dst_bytes = prod * di.elem_size;
    if ((total == 0) != (prod == 0)) { o.status = B200TFS_E_SHAPE; return; }
    if (total < prod) { o.status = B200TFS_E_SHAPE; return; }   // every element needs at least one byte
  } else {  // strings: unpacked on the host from msg_off/msg_len
    if (infer >= 0) {
      if (prod == 0 || o.n_strings % prod) { o.status = B200TFS_E_SHAPE; return; }
      set_dim(infer, (int64_t)(o.n_strings / prod)); prod = o.n_strings; o.flags |= B200TFS_OF_DIM_INFERRED;
    }
    o.n_elems = prod; o.dst_bytes = 0;
    if (o.n_strings != prod) { o.status = B200TFS_E_SHAPE; return; }
  }
}

B2_HD void spec_reset(b200tfs_model_spec& s) {
  s.name_off = 0; s.name_len = 0; s.signature_len = 0; s.signature_off = 0; s.label_off = 0; s.label_len = 0;
  s.has_version = 0; s.version = 0;
}

// ModelSpec (model.proto:9-33) in [c.p, c.end); repeated occurrences merge.
B2_HD void walk_model_spec(Cursor& c, b200tfs_model_spec& s) {
#pragma unroll 1
  while (c.p < c.end && !c.err) {
    const uint32_t tag = rd_tag(c);
    if (c.err) return;
    if (tag == tag_of(1, WT_LEN) || tag == tag_of(3, WT_LEN) || tag == tag_of(4, WT_LEN)) {
      uint32_t n;
      const uint32_t at = rd_string(c, &n);
      if (c.err) return;
      if ((tag >> 3) == 1) { s.name_off = at; s.name_len = n; }
      else if ((tag >> 3) == 3) { s.signature_off = at; s.signature_len = n; }
      else { s.label_off = at; s.label_len = n; s.has_version = 0; s.version = 0; }  // oneof: label displaces version
    } else if (tag == tag_of(2, WT_LEN)) {  // google.protobuf.Int64Value version
      const uint32_t n = rd_len(c);
      if (c.err) return;
      const uint32_t outer = c.end;
      c.end = c.p + n;
      if (!s.has_version) s.version = 0;
#pragma unroll 1
      while (c.p < c.end && !c.err) {
        const uint32_t t = rd_tag(c);
        if (c.err) break;
        if (t == tag_of(1, WT_VARINT)) s.version = (int64_t)rd_varint(c); else skip_field(c, t);
      }
      c.end = outer;
      if (c.err) return;
      s.has_version = 1; s.label_off = 0; s.label_len = 0;  // oneof: version displaces label
    } else skip_field(c, tag);
  }
}

B2_HD bool keys_equal(Cursor& c, const b200tfs_output& a, const b200tfs_output& b) {
  if (a.key_len != b.key_len) return false;
  const uint32_t pa = (uint32_t)a.key_off, pb = (uint32_t)b.key_off;
  for (uint32_t i = 0; i < a.key_len; ++i) if (rd8(c, pa + i) != rd8(c, pb + i)) return false;
  return true;
}

// One PredictResponse (predict.proto:30-40) occupying the cursor's record.
// outs needs max_outputs + 1 slots (the extra one is scratch for an entry whose key repeats).
// Returns the record status; *n_outs distinct keys.  B200TFS_E_SPILL: sp.used entries are needed, sp.cap were there.
B2_HD int walk_response(Cursor& c, int max_outputs, b200tfs_output* outs, int* n_outs, b200tfs_model_spec* spec, SpillArea& sp) {
  int n = 0;
  uint32_t seq = 0;
  sp.used = 0;
  spec_reset(*spec);
  *n_outs = 0;
#pragma unroll 1
  while (c.p < c.end && !c.err) {
    const uint32_t tag = rd_tag(c);
    if (c.err) break;
    if (tag == tag_of(1, WT_LEN)) {  // outputs map entry
      const uint32_t elen = rd_len(c);
      if (c.err) break;
      b200tfs_output& o = outs[n];  // parsed in place (slot n <= max_outputs); merged away below if the key repeats
      out_begin(o);
      WalkAux aux; aux_begin(aux, seq++);
      bool foreign = false;  // the entry itself carries a field that is not key/value
      const uint32_t outer = c.end;
      c.end = c.p + elen;
#pragma unroll 1
      while (c.p < c.end && !c.err) {
        const uint32_t t = rd_tag(c);
        if (c.err) break;
        if (t == tag_of(1, WT_LEN)) {
          uint32_t k;
          const uint32_t at = rd_string(c, &k);
          if (c.err) break;
          o.key_off = at; o.key_len = k;
        } else if (t == tag_of(2, WT_LEN)) {
          const uint32_t m = rd_len(c);
          if (c.err) break;
          o.msg_off = c.p; o.msg_len = m;
          const uint32_t inner = c.end;
          c.end = c.p + m;
          walk_tensor(c, o, sp, aux);
          c.end = inner;
        } else { skip_field(c, t); foreign = true; }
      }
      c.end = outer;
      if (c.err) break;
      // The runtime cannot keep unknown fields inside a map, so an entry that directly carries one
      // (incl. key/value with a mismatched wire type) stays an unknown field of the response and never
      // reaches the outputs map (pinned: tests/golden/decode.json "entry_with_foreign_field").
      if (foreign) continue;
      finalize_output(c, o, sp, aux);
      if (c.err) break;
      // duplicate key: the later entry replaces the earlier one
      int slot = -1;
      for (int i = 0; i < n; ++i) if (keys_equal(c, outs[i], o)) { slot = i; break; }
      if (slot >= 0) outs[slot] = o;
      else {
        if (n >= max_outputs) return B200TFS_E_SIZE;
        ++n;
      }
    } else if (tag == tag_of(2, WT_LEN)) {
      const uint32_t m = rd_len(c);
      if (c.err) break;
      const uint32_t outer = c.end;
      c.end = c.p + m;
      walk_model_spec(c, *spec);
      c.end = outer;
    } else skip_field(c, tag);
  }
  if (c.err) return c.err;
  if (sp.used > sp.cap) return B200TFS_E_SPILL;
  *n_outs = n;
  return B200TFS_OK;
}

// A bare TensorProto message (what tensor_proto_to_ndarray receives) occupying the cursor's record.
B2_HD int walk_tensor_proto(Cursor& c, b200tfs_output* out, SpillArea& sp) {
  out_begin(*out);
  WalkAux aux; aux_begin(aux, 0);
  sp.used = 0;
  out->msg_off = 0; out->msg_len = c.end;
  walk_tensor(c, *out, sp, aux);
  if (c.err) return c.err;
  if (sp.used > sp.cap) return B200TFS_E_SPILL;
  finalize_output(c, *out, sp, aux);
  return c.err ? c.err : B200TFS_OK;
}

}  // namespace b200tfs
