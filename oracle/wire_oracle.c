/* wire_oracle.c - CPU ORACLE.  TEST INFRASTRUCTURE ONLY: nothing in the product imports, links or
 * calls this file; only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
 * legs may (the product has no CPU path at all).
 *
 * A plain-C, scalar restatement of what the reference's Predict hot path puts on the wire and reads
 * back, pinned against vectors produced by the unmodified reference (tests/golden/, generated
 * by tests/golden/make_golden.py in the build container; tests/test_oracle.py replays every one of
 * them through this file).  Parity status: PINNED (encode: 43 TensorProto + 18 PredictRequest
 * vectors; decode: 58 PredictResponse vectors incl. every error class).
 *
 * Reference behaviour restated (paths relative to the reference checkout):
 *   tensor_serving_client/min_tfs_client/tensors.py:28-35   ndarray_to_tensor_proto: dtype enum, one
 *       Dim{size} per axis, values appended to the typed repeated field in C (ravel) order
 *   tensor_serving_client/min_tfs_client/tensors.py:17-25   write_values_to_tensor_proto: .item() per
 *       element -> float32 passes through a C double (sNaN quieted), ints through Python int
 *   tensor_serving_client/min_tfs_client/constants.py:13-29 dtype -> field table
 *   tensor_serving_client/min_tfs_client/requests.py:41-48  PredictRequest{model_spec{name,version},inputs}
 *   tensor_serving_client/min_tfs_client/tensors.py:38-46   extract_shape / tensor_proto_to_ndarray
 * The byte framing itself lives in the third-party protobuf runtime (pin protobuf>=3.8, reference
 * setup.py:102; the goldens were produced with 6.33.6/upb): proto3, fields in ascending number, zero
 * scalars elided, repeated scalars packed, map entries always carry key and value.
 *
 * Style: deliberately different from the product (csrc/): size-then-write emitters over a cursor,
 * and a decoder that materialises every repeated field as typed arrays instead of chunk tables.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORC_OK 0
#define ORC_E_DTYPE (-1)
#define ORC_E_SHAPE (-2)
#define ORC_E_PARSE (-4)
#define ORC_E_RANGE (-9)
#define ORC_E_KEY (-10)
#define ORC_E_RANK0 (-20) /* reshape() with no arguments: TypeError in the reference */
#define ORC_E_NOMEM (-21)

enum { DT_FLOAT = 1, DT_DOUBLE = 2, DT_INT32 = 3, DT_UINT8 = 4, DT_INT16 = 5, DT_INT8 = 6, DT_STRING = 7,
       DT_COMPLEX64 = 8, DT_INT64 = 9, DT_BOOL = 10, DT_BFLOAT16 = 14, DT_UINT16 = 17, DT_COMPLEX128 = 18,
       DT_HALF = 19, DT_UINT32 = 22, DT_UINT64 = 23 };

#define ORC_F_CONTENT 1   /* tensor_content instead of the typed field */
#define ORC_F_KEEP_SNAN 2 /* skip the float32 -> double -> float32 trip */

typedef struct {
  const void* data;   /* C-contiguous little-endian elements of src_dtype */
  int32_t src_dtype;
  int32_t wire_dtype; /* == src_dtype, or DT_FLOAT for HALF/BFLOAT16 sources */
  int32_t rank;
  int32_t flags;
  const int64_t* dims;
  const char* key;
  int64_t key_len;
} orc_tensor;

/* ------------------------------------------------------------------ emit helpers --------------- */
typedef struct { uint8_t* p; size_t n; } sink; /* p == NULL: count only */

static void put(sink* s, const void* src, size_t k) {
  if (s->p) memcpy(s->p + s->n, src, k);
  s->n += k;
}
static void put_byte(sink* s, unsigned b) { uint8_t x = (uint8_t)b; put(s, &x, 1); }
static void put_uvar(sink* s, uint64_t v) {
  do { unsigned b = v & 0x7F; v >>= 7; put_byte(s, b | (v ? 0x80 : 0)); } while (v);
}
static size_t uvar_size(uint64_t v) { size_t n = 1; while (v >>= 7) ++n; return n; }
static void put_tag(sink* s, unsigned field, unsigned wt) { put_uvar(s, ((uint64_t)field << 3) | wt); }

static int elem_size(int dt) {
  switch (dt) {
    case DT_FLOAT: case DT_INT32: case DT_UINT32: return 4;
    case DT_DOUBLE: case DT_INT64: case DT_UINT64: case DT_COMPLEX64: return 8;
    case DT_COMPLEX128: return 16;
    case DT_INT16: case DT_UINT16: case DT_HALF: case DT_BFLOAT16: return 2;
    case DT_INT8: case DT_UINT8: case DT_BOOL: return 1;
    default: return 0;
  }
}
static int field_of(int dt) {
  switch (dt) {
    case DT_FLOAT: return 5; case DT_DOUBLE: return 6;
    case DT_INT32: case DT_INT16: case DT_INT8: case DT_UINT8: case DT_UINT16: return 7;
    case DT_STRING: return 8; case DT_COMPLEX64: return 9; case DT_INT64: return 10; case DT_BOOL: return 11;
    case DT_COMPLEX128: return 12; case DT_HALF: case DT_BFLOAT16: return 13;
    case DT_UINT32: return 16; case DT_UINT64: return 17;
    default: return 0;
  }
}

/* float32 as the reference sees it: v.item() is a Python float (C double); protobuf stores it back
 * as a C float.  The double trip is what quiets signalling NaNs. */
static uint32_t through_double(uint32_t bits) {
  float f; volatile double d; float g; uint32_t out;
  memcpy(&f, &bits, 4);
  d = (double)f;
  g = (float)d;
  memcpy(&out, &g, 4);
  return out;
}

static uint32_t half_to_float_bits(uint16_t h) { /* exact widening, NaN payload kept */
  uint32_t sign = (uint32_t)(h & 0x8000) << 16, e = (h >> 10) & 0x1F, m = h & 0x3FF;
  if (e == 0) {
    if (!m) return sign;
    int sh = 0;
    while (!(m & 0x400)) { m <<= 1; ++sh; }
    return sign | (uint32_t)(127 - 15 - sh + 1) << 23 | (m & 0x3FF) << 13;
  }
  if (e == 31) return sign | 0x7F800000u | m << 13;
  return sign | (e + 112) << 23 | m << 13;
}

/* integer element i of a tensor as the int64 / uint64 the varint carries (int_val holds int32:
 * negatives are sign-extended to 64 bits, hence 10 bytes) */
static uint64_t int_elem(const void* data, int dt, uint64_t i) {
  switch (dt) {
    case DT_INT8: return (uint64_t)(int64_t)((const int8_t*)data)[i];
    case DT_INT16: return (uint64_t)(int64_t)((const int16_t*)data)[i];
    case DT_INT32: return (uint64_t)(int64_t)((const int32_t*)data)[i];
    case DT_INT64: return (uint64_t)((const int64_t*)data)[i];
    case DT_UINT8: return ((const uint8_t*)data)[i];
    case DT_UINT16: case DT_HALF: case DT_BFLOAT16: return ((const uint16_t*)data)[i];
    case DT_UINT32: return ((const uint32_t*)data)[i];
    default: return ((const uint64_t*)data)[i];
  }
}

static uint64_t count_elems(const orc_tensor* t) {
  uint64_t n = 1;
  for (int i = 0; i < t->rank; ++i) n *= (uint64_t)t->dims[i];
  return n;
}

/* packed body of the values field */
static void put_values(sink* s, const orc_tensor* t, uint64_t n) {
  const int content = t->flags & ORC_F_CONTENT;
  const int cast = t->src_dtype != t->wire_dtype; /* HALF / BFLOAT16 -> FLOAT */
  if (t->wire_dtype == DT_FLOAT) {
    for (uint64_t i = 0; i < n; ++i) {
      uint32_t w;
      if (!cast) w = ((const uint32_t*)t->data)[i];
      else if (t->src_dtype == DT_HALF) w = half_to_float_bits(((const uint16_t*)t->data)[i]);
      else w = (uint32_t)((const uint16_t*)t->data)[i] << 16;
      if (cast || (!content && !(t->flags & ORC_F_KEEP_SNAN))) w = through_double(w);
      put(s, &w, 4);
    }
    return;
  }
  if (content || t->wire_dtype == DT_DOUBLE || t->wire_dtype == DT_COMPLEX64 || t->wire_dtype == DT_COMPLEX128) {
    put(s, t->data, (size_t)(n * (uint64_t)elem_size(t->wire_dtype)));
    return;
  }
  if (t->wire_dtype == DT_BOOL) {
    for (uint64_t i = 0; i < n; ++i) put_byte(s, ((const uint8_t*)t->data)[i] ? 1 : 0);
    return;
  }
  for (uint64_t i = 0; i < n; ++i) put_uvar(s, int_elem(t->data, t->wire_dtype, i));
}

static void put_shape(sink* s, const orc_tensor* t) {
  for (int i = 0; i < t->rank; ++i) {
    uint64_t d = (uint64_t)t->dims[i];
    put_tag(s, 2, 2);
    if (d) { put_uvar(s, 1 + uvar_size(d)); put_tag(s, 1, 0); put_uvar(s, d); }
    else put_uvar(s, 0); /* Dim(size=0): empty sub-message */
  }
}

static int check_tensor(const orc_tensor* t) {
  if (!elem_size(t->src_dtype) || !elem_size(t->wire_dtype)) return ORC_E_DTYPE;
  if (t->src_dtype != t->wire_dtype && !(t->wire_dtype == DT_FLOAT && (t->src_dtype == DT_HALF || t->src_dtype == DT_BFLOAT16)))
    return ORC_E_DTYPE;
  for (int i = 0; i < t->rank; ++i) if (t->dims[i] < 0) return ORC_E_SHAPE;
  return ORC_OK;
}

static void put_tensor_proto(sink* s, const orc_tensor* t) {
  const uint64_t n = count_elems(t);
  sink c = {NULL, 0};
  put_tag(s, 1, 0); put_uvar(s, (uint64_t)t->wire_dtype);
  put_shape(&c, t);
  put_tag(s, 2, 2); put_uvar(s, c.n); put_shape(s, t); /* tensor_shape is always present (set in the constructor) */
  if (n) {
    sink v = {NULL, 0};
    put_values(&v, t, n);
    put_tag(s, (t->flags & ORC_F_CONTENT) ? 4 : (unsigned)field_of(t->wire_dtype), 2);
    put_uvar(s, v.n);
    put_values(s, t, n);
  }
}

/* Serialised TensorProto.  out == NULL: returns the size.  <0: error. */
int64_t orc_tensor_proto(const orc_tensor* t, uint8_t* out) {
  int rc = check_tensor(t);
  if (rc) return rc;
  sink s = {out, 0};
  put_tensor_proto(&s, t);
  return (int64_t)s.n;
}

/* deterministic map order of the protobuf (upb) runtime the goldens came from: bytewise over the
 * common prefix; when one key is a prefix of the other the LONGER one goes first */
static int upb_before(const orc_tensor* a, const orc_tensor* b) {
  size_t la = (size_t)a->key_len, lb = (size_t)b->key_len, m = la < lb ? la : lb;
  int c = memcmp(a->key, b->key, m);
  if (c) return c < 0;
  return la > lb;
}
void orc_order_upb(int n, const orc_tensor* ts, int32_t* perm) {
  for (int i = 0; i < n; ++i) perm[i] = i;
  for (int i = 1; i < n; ++i) { /* insertion sort: stable, n is small */
    int32_t x = perm[i];
    int j = i - 1;
    while (j >= 0 && upb_before(&ts[x], &ts[perm[j]])) { perm[j + 1] = perm[j]; --j; }
    perm[j + 1] = x;
  }
}

/* Serialised PredictRequest with the inputs in the order given.  out == NULL: size. */
int64_t orc_predict_request(const char* name, int64_t name_len, int has_version, int64_t version, int n,
                            const orc_tensor* inputs, uint8_t* out) {
  for (int i = 0; i < n; ++i) { int rc = check_tensor(&inputs[i]); if (rc) return rc; }
  sink s = {out, 0};
  /* model_spec: present even when empty, because requests.py:42 assigns into it */
  size_t vlen = version ? 1 + uvar_size((uint64_t)version) : 0;
  size_t spec = (name_len ? 1 + uvar_size((uint64_t)name_len) + (size_t)name_len : 0) + (has_version ? 2 + vlen : 0);
  put_tag(&s, 1, 2); put_uvar(&s, spec);
  if (name_len) { put_tag(&s, 1, 2); put_uvar(&s, (uint64_t)name_len); put(&s, name, (size_t)name_len); }
  if (has_version) {
    put_tag(&s, 2, 2); put_uvar(&s, vlen);
    if (version) { put_tag(&s, 1, 0); put_uvar(&s, (uint64_t)version); }
  }
  for (int i = 0; i < n; ++i) {
    const orc_tensor* t = &inputs[i];
    sink tp = {NULL, 0};
    put_tensor_proto(&tp, t);
    size_t entry = 1 + uvar_size((uint64_t)t->key_len) + (size_t)t->key_len + 1 + uvar_size(tp.n) + tp.n;
    put_tag(&s, 2, 2); put_uvar(&s, entry);
    put_tag(&s, 1, 2); put_uvar(&s, (uint64_t)t->key_len); put(&s, t->key, (size_t)t->key_len);
    put_tag(&s, 2, 2); put_uvar(&s, tp.n);
    put_tensor_proto(&s, t);
  }
  return (int64_t)s.n;
}

/* A PredictResponse the way tensorflow_model_server lays it out (outputs entries, then model_spec
 * {name, version, signature_name}); used to manufacture decode inputs at any size. */
int64_t orc_predict_response(const char* name, int64_t name_len, int64_t version, const char* sig, int64_t sig_len, int n,
                             const orc_tensor* outputs, uint8_t* out) {
  for (int i = 0; i < n; ++i) { int rc = check_tensor(&outputs[i]); if (rc) return rc; }
  sink s = {out, 0};
  for (int i = 0; i < n; ++i) {
    const orc_tensor* t = &outputs[i];
    sink tp = {NULL, 0};
    put_tensor_proto(&tp, t);
    size_t entry = 1 + uvar_size((uint64_t)t->key_len) + (size_t)t->key_len + 1 + uvar_size(tp.n) + tp.n;
    put_tag(&s, 1, 2); put_uvar(&s, entry);
    put_tag(&s, 1, 2); put_uvar(&s, (uint64_t)t->key_len); put(&s, t->key, (size_t)t->key_len);
    put_tag(&s, 2, 2); put_uvar(&s, tp.n);
    put_tensor_proto(&s, t);
  }
  size_t vlen = version ? 1 + uvar_size((uint64_t)version) : 0;
  size_t spec = (name_len ? 1 + uvar_size((uint64_t)name_len) + (size_t)name_len : 0) + 2 + vlen +
                (sig_len ? 1 + uvar_size((uint64_t)sig_len) + (size_t)sig_len : 0);
  put_tag(&s, 2, 2); put_uvar(&s, spec);
  if (name_len) { put_tag(&s, 1, 2); put_uvar(&s, (uint64_t)name_len); put(&s, name, (size_t)name_len); }
  put_tag(&s, 2, 2); put_uvar(&s, vlen);
  if (version) { put_tag(&s, 1, 0); put_uvar(&s, (uint64_t)version); }
  if (sig_len) { put_tag(&s, 3, 2); put_uvar(&s, (uint64_t)sig_len); put(&s, sig, (size_t)sig_len); }
  return (int64_t)s.n;
}

/* ------------------------------------------------------------------ decode --------------------- */
typedef struct { const uint8_t* p; const uint8_t* end; int bad; } rd;

static uint64_t get_uvar(rd* r) {
  uint64_t v = 0;
  for (int sh = 0; sh < 70; sh += 7) {
    if (r->p >= r->end) { r->bad = 1; return 0; }
    uint8_t b = *r->p++;
    if (sh < 64) v |= (uint64_t)(b & 0x7F) << sh;
    if (!(b & 0x80)) return v;
  }
  r->bad = 1;
  return 0;
}
static rd get_sub(rd* r) { /* length-delimited body */
  rd s = {r->p, r->p, 0};
  uint64_t n = get_uvar(r);
  if (r->bad || n > 0x7FFFFFFFu || n > (uint64_t)(r->end - r->p)) { r->bad = 1; s.bad = 1; return s; }
  s.p = r->p; s.end = r->p + n;
  r->p += n;
  return s;
}
static void skip_value(rd* r, uint64_t tag);
static void skip_group(rd* r, uint64_t field) {
  for (;;) {
    if (r->p >= r->end) { r->bad = 1; return; }
    const uint8_t* at = r->p;
    uint64_t t = get_uvar(r);
    if (r->bad) return;
    if (r->p - at > 5 || t > 0xFFFFFFFFu || !(t >> 3)) { r->bad = 1; return; }
    if ((t & 7) == 4) { if ((t >> 3) != field) r->bad = 1; return; }
    skip_value(r, t);
    if (r->bad) return;
  }
}
static void skip_value(rd* r, uint64_t tag) {
  switch (tag & 7) {
    case 0: (void)get_uvar(r); break;
    case 1: if (r->end - r->p < 8) r->bad = 1; else r->p += 8; break;
    case 2: (void)get_sub(r); break;
    case 3: skip_group(r, tag >> 3); break;
    case 5: if (r->end - r->p < 4) r->bad = 1; else r->p += 4; break;
    default: r->bad = 1;
  }
}
static uint64_t get_tag(rd* r) { /* at most 5 bytes, fits 32 bits, field number != 0 */
  const uint8_t* at = r->p;
  uint64_t t = get_uvar(r);
  if (!r->bad && (r->p - at > 5 || t > 0xFFFFFFFFu || !(t >> 3))) r->bad = 1;
  return t;
}
static int utf8_valid(const uint8_t* s, size_t n) {
  size_t i = 0;
  while (i < n) {
    uint32_t c = s[i], need, cp;
    if (c < 0x80) { ++i; continue; }
    if (c >= 0xC2 && c <= 0xDF) { need = 1; cp = c & 0x1F; }
    else if ((c & 0xF0) == 0xE0) { need = 2; cp = c & 0x0F; }
    else if (c >= 0xF0 && c <= 0xF4) { need = 3; cp = c & 0x07; }
    else return 0;
    if (n - i <= need) return 0;
    for (uint32_t k = 1; k <= need; ++k) { if ((s[i + k] & 0xC0) != 0x80) return 0; cp = cp << 6 | (s[i + k] & 0x3F); }
    if (need == 2 && (cp < 0x800 || (cp >= 0xD800 && cp <= 0xDFFF))) return 0;
    if (need == 3 && (cp < 0x10000 || cp > 0x10FFFF)) return 0;
    i += need + 1;
  }
  return 1;
}

/* growable typed arrays, one per TensorProto repeated field */
typedef struct { void* p; size_t n, cap, esz; } vec;
static int vec_push(vec* v, const void* x) {
  if (v->n == v->cap) {
    size_t c = v->cap ? v->cap * 2 : 64;
    void* q = realloc(v->p, c * v->esz);
    if (!q) return 0;
    v->p = q; v->cap = c;
  }
  memcpy((char*)v->p + v->n * v->esz, x, v->esz);
  ++v->n;
  return 1;
}

#define ORC_MAX_RANK 64
typedef struct {
  const uint8_t* key; size_t key_len;
  int32_t dtype; int32_t rank;
  int64_t dims[ORC_MAX_RANK];
  vec f32, f64, i32, i64, b8, h32, u32, u64, c64, c128; /* float_val double_val int_val int64_val bool_val half_val uint32_val uint64_val scomplex dcomplex */
  size_t n_strings, content_len;
  const uint8_t* content;
  const uint8_t* msg; size_t msg_len;
  int nomem;
} orc_out;

static void out_init(orc_out* o) {
  memset(o, 0, sizeof *o);
  o->f32.esz = 4; o->f64.esz = 8; o->i32.esz = 4; o->i64.esz = 8; o->b8.esz = 1; o->h32.esz = 4; o->u32.esz = 4; o->u64.esz = 8;
  o->c64.esz = 4; o->c128.esz = 8;
}
static void out_free(orc_out* o) {
  vec* vs[] = {&o->f32, &o->f64, &o->i32, &o->i64, &o->b8, &o->h32, &o->u32, &o->u64, &o->c64, &o->c128};
  for (size_t i = 0; i < sizeof vs / sizeof *vs; ++i) free(vs[i]->p);
}

static void read_shape(rd* r, orc_out* o) {
  while (r->p < r->end && !r->bad) {
    uint64_t t = get_tag(r);
    if (r->bad) return;
    if (t == (2 << 3 | 2)) {
      rd d = get_sub(r);
      if (r->bad) return;
      int64_t size = 0;
      while (d.p < d.end && !d.bad) {
        uint64_t dt = get_tag(&d);
        if (d.bad) break;
        if (dt == (1 << 3 | 0)) size = (int64_t)get_uvar(&d);
        else if (dt == (2 << 3 | 2)) { rd nm = get_sub(&d); if (!d.bad && !utf8_valid(nm.p, (size_t)(nm.end - nm.p))) d.bad = 1; }
        else skip_value(&d, dt);
      }
      if (d.bad) { r->bad = 1; return; }
      if (o->rank < ORC_MAX_RANK) o->dims[o->rank++] = size; else { r->bad = 1; return; }
    } else skip_value(r, t);
  }
}

/* one occurrence of a repeated scalar field: packed run (wire type 2) or a single element */
static void read_scalars(rd* r, orc_out* o, unsigned field, unsigned wt) {
  vec* v; int kind; /* 0 varint, 4 fixed32, 8 fixed64 */
  switch (field) {
    case 5: v = &o->f32; kind = 4; break;  case 6: v = &o->f64; kind = 8; break;
    case 7: v = &o->i32; kind = 0; break;  case 9: v = &o->c64; kind = 4; break;
    case 10: v = &o->i64; kind = 0; break; case 11: v = &o->b8; kind = 0; break;
    case 12: v = &o->c128; kind = 8; break; case 13: v = &o->h32; kind = 0; break;
    case 16: v = &o->u32; kind = 0; break; default: v = &o->u64; kind = 0; break;
  }
  rd body;
  if (wt == 2) { body = get_sub(r); if (r->bad) return; }
  else {
    unsigned want = kind == 4 ? 5 : kind == 8 ? 1 : 0;
    if (wt != want) { skip_value(r, (uint64_t)field << 3 | wt); return; } /* mismatched wire type: unknown field */
    body.p = r->p; body.bad = 0;
    if (kind) { if ((size_t)(r->end - r->p) < (size_t)kind) { r->bad = 1; return; } body.end = r->p + kind; r->p += kind; }
    else { (void)get_uvar(r); if (r->bad) return; body.end = r->p; }
  }
  if (kind && (size_t)(body.end - body.p) % (size_t)kind) { r->bad = 1; return; }
  while (body.p < body.end) {
    if (kind == 4) { uint32_t w; memcpy(&w, body.p, 4); body.p += 4; if (!vec_push(v, &w)) o->nomem = 1; }
    else if (kind == 8) { uint64_t w; memcpy(&w, body.p, 8); body.p += 8; if (!vec_push(v, &w)) o->nomem = 1; }
    else {
      uint64_t x = get_uvar(&body);
      if (body.bad) { r->bad = 1; return; }
      if (field == 7 || field == 13) { int32_t y = (int32_t)(uint32_t)x; if (!vec_push(v, &y)) o->nomem = 1; }       /* int32 fields truncate */
      else if (field == 16) { uint32_t y = (uint32_t)x; if (!vec_push(v, &y)) o->nomem = 1; }
      else if (field == 11) { uint8_t y = x != 0; if (!vec_push(v, &y)) o->nomem = 1; }
      else if (!vec_push(v, &x)) o->nomem = 1;
    }
  }
}

/* resource_handle_val / variant_val are never read on this path, but the runtime parses them, so
 * malformed bytes inside them fail the message: validate structure recursively (schemas:
 * resource_handle.proto:16-42, tensor.proto:87-94). */
static void check_shape(rd* r);
static void check_nested_tensor(rd* r, int depth);
static void check_string(rd* r) { rd s = get_sub(r); if (!r->bad && !utf8_valid(s.p, (size_t)(s.end - s.p))) r->bad = 1; }
static void check_shape(rd* r) {
  while (r->p < r->end && !r->bad) {
    uint64_t t = get_tag(r);
    if (r->bad) return;
    if (t == (2 << 3 | 2)) {
      rd d = get_sub(r);
      if (r->bad) return;
      while (d.p < d.end && !d.bad) {
        uint64_t dt = get_tag(&d);
        if (d.bad) break;
        if (dt == (2 << 3 | 2)) check_string(&d); else skip_value(&d, dt);
      }
      if (d.bad) r->bad = 1;
    } else skip_value(r, t);
  }
}
static void check_resource(rd* r) {
  while (r->p < r->end && !r->bad) {
    uint64_t t = get_tag(r);
    if (r->bad) return;
    unsigned f = (unsigned)(t >> 3), wt = (unsigned)(t & 7);
    if (wt == 2 && (f == 1 || f == 2 || f == 3 || f == 5)) check_string(r);
    else if (wt == 2 && f == 6) {
      rd d = get_sub(r);
      if (r->bad) return;
      while (d.p < d.end && !d.bad) {
        uint64_t dt = get_tag(&d);
        if (d.bad) break;
        if (dt == (2 << 3 | 2)) { rd s = get_sub(&d); if (!d.bad) { check_shape(&s); if (s.bad) d.bad = 1; } }
        else skip_value(&d, dt);
      }
      if (d.bad) r->bad = 1;
    } else skip_value(r, t);
  }
}
static void check_variant(rd* r, int depth) {
  while (r->p < r->end && !r->bad) {
    uint64_t t = get_tag(r);
    if (r->bad) return;
    if (t == (1 << 3 | 2)) check_string(r);
    else if (t == (3 << 3 | 2)) { rd s = get_sub(r); if (!r->bad) { check_nested_tensor(&s, depth + 1); if (s.bad) r->bad = 1; } }
    else skip_value(r, t);
  }
}
static void check_nested_tensor(rd* r, int depth) {
  if (depth > 64) { r->bad = 1; return; }
  while (r->p < r->end && !r->bad) {
    uint64_t t = get_tag(r);
    if (r->bad) return;
    unsigned f = (unsigned)(t >> 3), wt = (unsigned)(t & 7);
    if (wt != 2) { skip_value(r, t); continue; }
    rd s = get_sub(r);
    if (r->bad) return;
    size_t n = (size_t)(s.end - s.p);
    if (f == 2) check_shape(&s);
    else if (f == 14) check_resource(&s);
    else if (f == 15) check_variant(&s, depth);
    else if (f == 5 || f == 9) { if (n % 4) s.bad = 1; }
    else if (f == 6 || f == 12) { if (n % 8) s.bad = 1; }
    else if (f == 7 || f == 10 || f == 11 || f == 13 || f == 16 || f == 17) { if (n && (s.end[-1] & 0x80)) s.bad = 1; }
    if (s.bad) r->bad = 1;
  }
}

static void read_tensor(rd* r, orc_out* o) {
  while (r->p < r->end && !r->bad) {
    uint64_t t = get_tag(r);
    if (r->bad) return;
    unsigned field = (unsigned)(t >> 3), wt = (unsigned)(t & 7);
    if (field == 1 && wt == 0) o->dtype = (int32_t)(uint32_t)get_uvar(r);
    else if (field == 2 && wt == 2) { rd s = get_sub(r); if (r->bad) return; read_shape(&s, o); if (s.bad) r->bad = 1; }
    else if (field == 4 && wt == 2) { rd s = get_sub(r); if (r->bad) return; o->content = s.p; o->content_len = (size_t)(s.end - s.p); }
    else if (field == 8 && wt == 2) { (void)get_sub(r); o->n_strings++; }
    else if (field == 14 && wt == 2) { rd s = get_sub(r); if (r->bad) return; check_resource(&s); if (s.bad) r->bad = 1; }
    else if (field == 15 && wt == 2) { rd s = get_sub(r); if (r->bad) return; check_variant(&s, 0); if (s.bad) r->bad = 1; }
    else if ((field >= 5 && field <= 7) || (field >= 9 && field <= 13) || field == 16 || field == 17) read_scalars(r, o, field, wt);
    else skip_value(r, t);
  }
}

/* float32 read back: float_val elements become Python floats (double) and are written into a
 * float32 numpy array: the same double trip as on encode */
static int64_t prod_dims(const orc_out* o, int* infer_at) {
  int64_t prod = 1; *infer_at = -1;
  for (int i = 0; i < o->rank; ++i) {
    if (o->dims[i] == -1 && *infer_at < 0) { *infer_at = i; continue; }
    if (o->dims[i] < 0) return -1;
    prod *= o->dims[i];
  }
  return prod;
}

/* Number of elements numpy would hold for this output before reshape, -1 if dtype is unmapped. */
static int64_t element_count(const orc_out* o) {
  switch (o->dtype) {
    case DT_FLOAT: return (int64_t)o->f32.n;   case DT_DOUBLE: return (int64_t)o->f64.n;
    case DT_INT32: case DT_INT16: case DT_INT8: case DT_UINT8: case DT_UINT16: return (int64_t)o->i32.n;
    case DT_INT64: return (int64_t)o->i64.n;   case DT_BOOL: return (int64_t)o->b8.n;
    case DT_HALF: case DT_BFLOAT16: return (int64_t)o->h32.n;
    case DT_UINT32: return (int64_t)o->u32.n;  case DT_UINT64: return (int64_t)o->u64.n;
    case DT_COMPLEX64: return (int64_t)o->c64.n / 2; case DT_COMPLEX128: return (int64_t)o->c128.n / 2;
    case DT_STRING: return (int64_t)o->n_strings;
    default: return -1;
  }
}

/* ---- flat C interface for ctypes -------------------------------------------------------------- */
#define ORC_MAX_OUT 64
typedef struct {
  int64_t key_off, key_len;  /* into the wire */
  int32_t dtype, rank, status, pad;
  int64_t dims[ORC_MAX_RANK];
  int64_t n_elems;           /* after reshape */
  int64_t msg_off, msg_len;  /* the TensorProto sub-message */
} orc_desc;

typedef struct {
  int64_t name_off, name_len, sig_off, sig_len, label_off, label_len, version;
  int32_t has_version, pad;
} orc_spec;

typedef struct {
  const uint8_t* wire;
  int n;
  orc_out outs[ORC_MAX_OUT];
} orc_parsed;

void orc_free(orc_parsed* p) {
  if (!p) return;
  for (int i = 0; i < p->n; ++i) out_free(&p->outs[i]);
  free(p);
}

static void settle(const orc_out* o, orc_desc* d) {
  int infer;
  d->dtype = o->dtype; d->rank = o->rank; d->status = ORC_OK;
  memcpy(d->dims, o->dims, sizeof d->dims);
  int64_t cnt = element_count(o);
  if (cnt < 0) { d->status = ORC_E_KEY; return; }
  int64_t prod = prod_dims(o, &infer);
  if (prod < 0) { d->status = ORC_E_SHAPE; return; }
  if (infer >= 0) {
    if (prod == 0 || cnt % prod) { d->status = ORC_E_SHAPE; return; }
    d->dims[infer] = cnt / prod; prod = cnt;
  }
  if (cnt != prod) { d->status = ORC_E_SHAPE; return; }
  d->n_elems = prod;
  if (o->rank == 0) d->status = ORC_E_RANK0;
}

/* Parse one PredictResponse.  Returns a handle (free with orc_free) or NULL on malformed input. */
orc_parsed* orc_parse_response(const uint8_t* wire, int64_t len, orc_desc* descs, int32_t* n_out, orc_spec* spec) {
  orc_parsed* P = (orc_parsed*)calloc(1, sizeof *P);
  if (!P) return NULL;
  P->wire = wire;
  memset(spec, 0, sizeof *spec);
  rd r = {wire, wire + len, 0};
  while (r.p < r.end && !r.bad) {
    uint64_t t = get_tag(&r);
    if (r.bad) break;
    if (t == (1 << 3 | 2)) {
      rd e = get_sub(&r);
      if (r.bad) break;
      orc_out o; out_init(&o);
      int foreign = 0; /* an entry that itself holds an unknown field is kept as an unknown field of the
                          response by the runtime and never enters the map */
      while (e.p < e.end && !e.bad) {
        uint64_t et = get_tag(&e);
        if (e.bad) break;
        if (et == (1 << 3 | 2)) {
          rd k = get_sub(&e);
          if (e.bad) break;
          if (!utf8_valid(k.p, (size_t)(k.end - k.p))) { e.bad = 1; break; }
          o.key = k.p; o.key_len = (size_t)(k.end - k.p);
        } else if (et == (2 << 3 | 2)) {
          rd v = get_sub(&e);
          if (e.bad) break;
          o.msg = v.p; o.msg_len = (size_t)(v.end - v.p);
          read_tensor(&v, &o);
          if (v.bad) e.bad = 1;
        } else { skip_value(&e, et); foreign = 1; }
      }
      if (e.bad || o.nomem) { out_free(&o); r.bad = 1; break; }
      if (foreign) { out_free(&o); continue; }
      int slot = -1;
      for (int i = 0; i < P->n; ++i)
        if (P->outs[i].key_len == o.key_len && (!o.key_len || !memcmp(P->outs[i].key, o.key, o.key_len))) slot = i;
      if (slot >= 0) { out_free(&P->outs[slot]); P->outs[slot] = o; }
      else if (P->n < ORC_MAX_OUT) P->outs[P->n++] = o;
      else { out_free(&o); r.bad = 1; break; }
    } else if (t == (2 << 3 | 2)) {
      rd m = get_sub(&r);
      if (r.bad) break;
      while (m.p < m.end && !m.bad) {
        uint64_t mt = get_tag(&m);
        if (m.bad) break;
        if (mt == (1 << 3 | 2) || mt == (3 << 3 | 2) || mt == (4 << 3 | 2)) {
          rd sv = get_sub(&m);
          if (m.bad) break;
          if (!utf8_valid(sv.p, (size_t)(sv.end - sv.p))) { m.bad = 1; break; }
          int64_t off = sv.p - wire, n = sv.end - sv.p;
          if ((mt >> 3) == 1) { spec->name_off = off; spec->name_len = n; }
          else if ((mt >> 3) == 3) { spec->sig_off = off; spec->sig_len = n; }
          else { spec->label_off = off; spec->label_len = n; spec->has_version = 0; spec->version = 0; }
        } else if (mt == (2 << 3 | 2)) {
          rd iv = get_sub(&m);
          if (m.bad) break;
          if (!spec->has_version) spec->version = 0;
          while (iv.p < iv.end && !iv.bad) {
            uint64_t vt = get_tag(&iv);
            if (iv.bad) break;
            if (vt == (1 << 3 | 0)) spec->version = (int64_t)get_uvar(&iv); else skip_value(&iv, vt);
          }
          if (iv.bad) { m.bad = 1; break; }
          spec->has_version = 1; spec->label_off = 0; spec->label_len = 0;
        } else skip_value(&m, mt);
      }
      if (m.bad) r.bad = 1;
    } else skip_value(&r, t);
  }
  if (r.bad) { orc_free(P); return NULL; }
  *n_out = P->n;
  for (int i = 0; i < P->n; ++i) {
    orc_desc* d = &descs[i];
    memset(d, 0, sizeof *d);
    d->key_off = P->outs[i].key ? P->outs[i].key - wire : 0;
    d->key_len = (int64_t)P->outs[i].key_len;
    d->msg_off = P->outs[i].msg ? P->outs[i].msg - wire : 0;
    d->msg_len = (int64_t)P->outs[i].msg_len;
    settle(&P->outs[i], d);
  }
  return P;
}

/* A bare TensorProto. */
orc_parsed* orc_parse_tensor(const uint8_t* wire, int64_t len, orc_desc* desc) {
  orc_parsed* P = (orc_parsed*)calloc(1, sizeof *P);
  if (!P) return NULL;
  P->wire = wire;
  rd r = {wire, wire + len, 0};
  out_init(&P->outs[0]);
  P->n = 1;
  read_tensor(&r, &P->outs[0]);
  if (r.bad || P->outs[0].nomem) { orc_free(P); return NULL; }
  memset(desc, 0, sizeof *desc);
  desc->msg_off = 0; desc->msg_len = len;
  settle(&P->outs[0], desc);
  return P;
}

/* Write output i as `dtype` elements into dst (n_elems of them).  half_mode: 0 = TF (bit patterns),
 * 1 = the reference's quirk (half_val integers are VALUES converted to float16). */
static uint16_t int_to_half(int32_t v) { /* round-to-nearest-even, overflow -> inf */
  uint16_t sign = 0;
  uint32_t a;
  if (v < 0) { sign = 0x8000; a = (uint32_t)(-(int64_t)v); } else a = (uint32_t)v;
  if (!a) return sign;
  int e = 31;
  while (!(a >> e)) --e;
  if (e > 15) return sign | 0x7C00;
  uint32_t m; /* 11 significant bits incl. hidden */
  if (e <= 10) m = a << (10 - e);
  else {
    int sh = e - 10;
    uint32_t rem = a & ((1u << sh) - 1), half = 1u << (sh - 1);
    m = a >> sh;
    if (rem > half || (rem == half && (m & 1))) ++m;
    if (m >> 11) { m >>= 1; ++e; if (e > 15) return sign | 0x7C00; }
  }
  return sign | (uint16_t)((e + 15) << 10) | (uint16_t)(m & 0x3FF);
}

int32_t orc_write_output(const orc_parsed* P, int i, int half_mode, void* dst) {
  const orc_out* o = &P->outs[i];
  switch (o->dtype) {
    case DT_FLOAT: for (size_t k = 0; k < o->f32.n; ++k) ((uint32_t*)dst)[k] = through_double(((uint32_t*)o->f32.p)[k]); return ORC_OK;
    case DT_DOUBLE: memcpy(dst, o->f64.p, o->f64.n * 8); return ORC_OK;
    case DT_COMPLEX64: memcpy(dst, o->c64.p, o->c64.n * 4); return ORC_OK;
    case DT_COMPLEX128: memcpy(dst, o->c128.p, o->c128.n * 8); return ORC_OK;
    case DT_INT64: memcpy(dst, o->i64.p, o->i64.n * 8); return ORC_OK;
    case DT_UINT64: memcpy(dst, o->u64.p, o->u64.n * 8); return ORC_OK;
    case DT_UINT32: memcpy(dst, o->u32.p, o->u32.n * 4); return ORC_OK;
    case DT_INT32: memcpy(dst, o->i32.p, o->i32.n * 4); return ORC_OK;
    case DT_BOOL: memcpy(dst, o->b8.p, o->b8.n); return ORC_OK;
    case DT_INT16: for (size_t k = 0; k < o->i32.n; ++k) { int32_t v = ((int32_t*)o->i32.p)[k]; if (v < -32768 || v > 32767) return ORC_E_RANGE; ((int16_t*)dst)[k] = (int16_t)v; } return ORC_OK;
    case DT_INT8: for (size_t k = 0; k < o->i32.n; ++k) { int32_t v = ((int32_t*)o->i32.p)[k]; if (v < -128 || v > 127) return ORC_E_RANGE; ((int8_t*)dst)[k] = (int8_t)v; } return ORC_OK;
    case DT_UINT16: for (size_t k = 0; k < o->i32.n; ++k) { int32_t v = ((int32_t*)o->i32.p)[k]; if (v < 0 || v > 65535) return ORC_E_RANGE; ((uint16_t*)dst)[k] = (uint16_t)v; } return ORC_OK;
    case DT_UINT8: for (size_t k = 0; k < o->i32.n; ++k) { int32_t v = ((int32_t*)o->i32.p)[k]; if (v < 0 || v > 255) return ORC_E_RANGE; ((uint8_t*)dst)[k] = (uint8_t)v; } return ORC_OK;
    case DT_HALF: case DT_BFLOAT16:
      for (size_t k = 0; k < o->h32.n; ++k) {
        int32_t v = ((int32_t*)o->h32.p)[k];
        ((uint16_t*)dst)[k] = (half_mode && o->dtype == DT_HALF) ? int_to_half(v) : (uint16_t)v;
      }
      return ORC_OK;
    default: return ORC_E_KEY;
  }
}

/* ------------------------------------------------------------------ 16-bit float conversions --- */
/* float32 bits -> float16 (to_bf16 = 0) or bfloat16 (1) bits as `tensor_proto_to_ndarray(...).astype(...)` gives them:
 * the float32 was read back through a C double, so a NaN is quiet before it is narrowed (numpy keeps the top ten payload
 * bits for float16, ml_dtypes writes the canonical quiet NaN for bfloat16, sign kept by both).  Everything else rounds
 * to nearest even: integer arithmetic only, so the reference does not share the rounding hardware it checks. */
static uint16_t narrow_bits(uint32_t w, int to_bf16) {
  const int mb = to_bf16 ? 7 : 10, bias = to_bf16 ? 127 : 15; /* kept mantissa bits, exponent bias */
  const uint32_t inf = to_bf16 ? 0x7F80u : 0x7C00u;
  const uint32_t sign = (w >> 16) & 0x8000u;
  int e = (int)((w >> 23) & 0xFF);
  uint32_t sig = w & 0x7FFFFFu;
  if (e == 0xFF) {
    if (!sig) return (uint16_t)(sign | inf);
    w |= 0x400000u;
    return (uint16_t)(to_bf16 ? sign | 0x7FC0u : sign | 0x7E00u | ((w >> 13) & 0x3FFu));
  }
  if (!e && !sig) return (uint16_t)sign;
  /* value = sig * 2^(k - 23) with 2^23 <= sig < 2^24 */
  int k = e - 127;
  if (e) sig |= 0x800000u;
  else { k = -126; while (!(sig & 0x800000u)) { sig <<= 1; --k; } }
  /* quantum of the result: 2^(t - mb), t = k clamped to the smallest normal exponent (subnormal results) */
  int t = k < 1 - bias ? 1 - bias : k;
  int sh = 23 + t - k - mb; /* >= 23 - mb > 0 */
  if (sh > 25) sh = 25;     /* sig < 2^24 <= half: rounds to zero either way */
  uint32_t q = sig >> sh, rem = sig & ((1u << sh) - 1), half = 1u << (sh - 1);
  if (rem > half || (rem == half && (q & 1))) ++q;
  /* biased exponent t + bias over q's implicit bit: a carry out of the mantissa moves into the exponent, a subnormal q
   * that rounds up to 2^mb becomes the smallest normal */
  uint32_t mag = ((uint32_t)(t + bias - 1) << mb) + q;
  if (mag >= inf) mag = inf;
  return (uint16_t)(sign | mag);
}

void orc_narrow_f32(const uint32_t* src, uint16_t* dst, int64_t n, int to_bf16) {
  for (int64_t i = 0; i < n; ++i) dst[i] = narrow_bits(src[i], to_bf16);
}

/* float16 / bfloat16 bits -> float32 bits as the reference puts them on the wire for wire_dtype DT_FLOAT (put_values) */
void orc_widen_16(const uint16_t* src, uint32_t* dst, int64_t n, int from_bf16) {
  for (int64_t i = 0; i < n; ++i)
    dst[i] = through_double(from_bf16 ? (uint32_t)src[i] << 16 : half_to_float_bits(src[i]));
}

/* DT_HALF half_val integers read as values (the reference's quirk, orc_write_output with half_mode 1) */
void orc_int_to_half(const int32_t* src, uint16_t* dst, int64_t n) {
  for (int64_t i = 0; i < n; ++i) dst[i] = int_to_half(src[i]);
}

/* typed values present for output i (complex: pairs), whatever the shape says; -1 if the dtype has no typed field */
int64_t orc_value_count(const orc_parsed* P, int i) { return element_count(&P->outs[i]); }
int64_t orc_content_len(const orc_parsed* P, int i) { return (int64_t)P->outs[i].content_len; }
int64_t orc_content_off(const orc_parsed* P, int i) { return P->outs[i].content ? P->outs[i].content - P->wire : 0; }
