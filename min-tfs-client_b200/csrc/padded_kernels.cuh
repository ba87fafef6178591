// padded_kernels.cuh - b200tfs_decode_padded: a batch of PredictResponses into one padded tensor per requested key (plan.h
// PaddedPlan; the host side is in codec_host.cpp).  Included by kernels.cu inside namespace b200tfs, after concat_plan_kernel.
//
//   padded_plan_kernel  one CTA.  Per key: concat_plan_kernel's pass A (plan_key_reference), then every record against the first
//                       record that decoded the key (dtype, rank) and against the destination's trailing dims, a block scan of
//                       dims[0] into first rows, one PadDesc per (record, key) and the single-launch decode's table for the
//                       varint tail.  Nothing waits on another CTA: a replayed graph re-plans rows and trailing dims.
//                       padded_plan_strings_kernel: the same with DT_STRING keys placed too (their kernels: at the end of this file).
//   padded_emit_kernel  destination-major: every CTA takes chunks of kPadChunkBytes of a key's used rows, finds the record of
//                       each row by binary search over the first rows and writes whole 16-byte vectors of values and pads, so
//                       every destination byte is written once.  Packed-varint keys: the pads only (vdec_emit_padded_kernel
//                       writes their values).

// byte j of the record's value stream (its runs in wire order; a run of count > 1 is a row of pieces `stride` bytes apart)
__device__ __forceinline__ uint8_t pad_src_byte(const PadDesc& d, uint64_t j) {
  for (uint32_t q = 0; q < d.n_runs; ++q) {
    const b200tfs_run& rn = d.runs[q];
    const uint64_t rb = (uint64_t)rn.len * rn.count;
    if (j < rb) return d.rec[rn.off + (rn.count > 1 ? (j / rn.len) * rn.stride + j % rn.len : j)];
    j -= rb;
  }
  return 0;
}

// `nb` (<= 8) bytes of the value stream from byte j, little-endian
__device__ __forceinline__ uint64_t pad_src_bytes(const PadDesc& d, uint64_t j, uint32_t nb) {
  uint64_t v = 0;
  if (d.n_runs && d.runs[0].count == 1 && j + nb <= d.runs[0].len) {   // the common case: one packed occurrence
    const uint8_t* p = d.rec + d.runs[0].off + j;
    for (uint32_t i = 0; i < nb; ++i) v |= (uint64_t)p[i] << (8 * i);
  } else {
    for (uint32_t i = 0; i < nb; ++i) v |= (uint64_t)pad_src_byte(d, j + i) << (8 * i);
  }
  return v;
}

// the last record whose first row is <= row (records without rows share their first row with the next one)
__device__ __forceinline__ uint32_t pad_find_rec(const uint64_t* fr, uint32_t n, uint64_t row) {
  uint32_t lo = 0, hi = n;
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) >> 1;
    if (fr[mid] <= row) lo = mid; else hi = mid;
  }
  return lo;
}

// kStrings: DT_STRING keys get rows too (b200tfs_decode_padded_strings): 8 bytes of int64 offsets per position and one entry
// behind the rows, no emit chunks; the pad_str_* kernels below fill them.  Without it they are left to the host.
template <bool kStrings>
__device__ __forceinline__ void padded_plan_body(const PaddedPlan& pp) {
  __shared__ unsigned long long warp_sum[kConcatPlanThreads / 32];
  __shared__ uint32_t ref_rec;
  __shared__ unsigned long long first_over;   // first row of the first record whose rows pass dst_cap
  const ConcatPlan& cp = pp.cp;
  const uint32_t n = cp.n, nk = cp.n_keys;
  uint64_t chunks = 0;
  for (uint32_t k = 0; k < nk; ++k) {
    const PadKeyDev& key = pp.keys[k];
    if (threadIdx.x == 0) first_over = ~0ull;
    const b200tfs_output* ro = plan_key_reference(cp, key.k.key, key.k.key_len, k, &ref_rec);
    const int32_t dtype = ro ? ro->dtype : 0, rank = key.rank;
    const DtypeInfo di = dtype_info(dtype);
    const bool narrow = tpl_narrows(cp.cast, dtype), varint = di.kind == VK_VARINT || di.kind == VK_BOOL;
    const bool str = kStrings && di.kind == VK_STRING;
    const uint32_t esz = str ? 8u : narrow ? 2u : di.elem_size;
    uint64_t row_elems = 1;
    for (int32_t a = 1; a < rank && a < B200TFS_MAX_RANK; ++a) row_elems *= (uint64_t)key.dims[a];
    const uint64_t pitch = row_elems * esz;
    uint64_t row_carry = 0;
    for (uint32_t r0 = 0; r0 < n; r0 += kConcatPlanThreads) {      // uniform trip count: the scan has barriers inside
      const uint32_t r = r0 + threadIdx.x;
      int32_t st = B200TFS_E_ARG;
      const b200tfs_output* o = nullptr;
      uint64_t rows = 0;
      if (r < n) {
        st = cp.kst[(size_t)r * nk + k];
        const int32_t m = cp.match[(size_t)r * nk + k];
        if (m >= 0) o = cp.outs + (size_t)r * cp.out_stride + m;
        if (st == B200TFS_OK) {
          if (o->dtype != ro->dtype) st = B200TFS_E_DTYPE;
          else if (o->rank != ro->rank || o->rank != rank) st = B200TFS_E_SHAPE;
          else for (int32_t a = 1; a < o->rank; ++a) if (o->dims[a] > key.dims[a]) st = B200TFS_E_SIZE;
        }
        if (st == B200TFS_OK) {
          const uint32_t kind = dtype_info(o->dtype).kind;
          // strings are decoded on the host (kStrings: by the string kernels); the emit reads the inline runs only; the varint
          // decode takes packed occurrences only
          if ((kind == VK_STRING && !kStrings) || (o->flags & B200TFS_OF_SPILLED) || o->n_inline != (uint32_t)o->n_runs)
            st = B200TFS_E_NONCANONICAL;
          if (kind == VK_VARINT || kind == VK_BOOL) {
            if (o->flags & B200TFS_OF_UNPACKED) st = B200TFS_E_NONCANONICAL;
            for (int32_t q = 0; q < o->n_runs && q < B200TFS_MAX_RUNS; ++q) if (o->runs[q].count != 1) st = B200TFS_E_NONCANONICAL;
          }
        }
        if (st == B200TFS_OK) rows = (uint64_t)o->dims[0];
      }
      const uint64_t first = concat_scan(rows, row_carry, warp_sum);
      if (r < n) {
        if (st == B200TFS_OK && rows && (first + rows) * pitch + (str ? 8u : 0u) > key.k.cap) {   // strings: the entry behind
          st = B200TFS_E_SIZE;
          atomicMin(&first_over, (unsigned long long)first);
        }
        const bool placed = st == B200TFS_OK;
        PadDesc d{};
        if (o) {
          d.n_runs = min(o->n_inline, (uint32_t)B200TFS_MAX_RUNS);
          for (uint32_t q = 0; q < d.n_runs; ++q) d.runs[q] = o->runs[q];
          for (int32_t a = 0; a < o->rank && a < B200TFS_MAX_RANK; ++a) d.dims[a] = o->dims[a];
        }
        d.rec = cp.w + cp.rec_off[r];
        d.first_row = first;
        d.rows = placed ? rows : 0;
        pp.desc[(size_t)r * nk + k] = d;
        pp.first_row[(size_t)k * n + r] = first;
        b200tfs_output v{};
        if (o) v = *o;
        v.status = st;
        v.dst_off = (uint64_t)(uintptr_t)(key.k.dst + first * pitch);
        v.dst_bytes = placed ? rows * pitch : 0;
        cp.vouts[(size_t)r * kFusedMaxOutputs + k] = v;
        if (k == 0) { cp.vn_outs[r] = (int32_t)nk; cp.vrec_status[r] = B200TFS_OK; }
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      const uint64_t used = min((uint64_t)row_carry, (uint64_t)first_over);
      PadKeyOut ko{};
      ko.rows = used; ko.pitch = pitch; ko.chunk0 = chunks;
      ko.row_elems = (uint32_t)row_elems; ko.esz = esz; ko.src_esz = di.elem_size; ko.op = tpl_move_op(cp.cast, dtype);
      ko.varint = varint ? 1u : 0u;
      ko.str = str ? 1u : 0u;
      pp.kout[k] = ko;
      if (!str) chunks += (used * pitch + kPadChunkBytes - 1) / kPadChunkBytes;
    }
  }
  if (threadIdx.x == 0) { PadKeyOut end{}; end.chunk0 = chunks; pp.kout[nk] = end; }
}

__global__ void __launch_bounds__(kConcatPlanThreads) padded_plan_kernel(const __grid_constant__ PaddedPlan pp) { padded_plan_body<false>(pp); }
__global__ void __launch_bounds__(kConcatPlanThreads) padded_plan_strings_kernel(const __grid_constant__ PaddedPlan pp) {
  padded_plan_body<true>(pp);
}

// one 16-byte vector of key k's destination, at byte b (< used) of it: ESZ-byte elements, values and pads
template <uint32_t ESZ>
__device__ __forceinline__ void pad_emit_vec(const PaddedPlan& pp, const PadKeyDev& key, const PadKeyOut& ko, uint32_t k, uint64_t b,
                                             uint64_t used) {
  constexpr uint32_t M = 16 / ESZ;
  const uint32_t n = pp.cp.n, nk = pp.cp.n_keys;
  const uint64_t* fr = pp.first_row + (size_t)k * n;
  const uint64_t* pw = reinterpret_cast<const uint64_t*>(key.pad);
  uint32_t w[4] = {0u, 0u, 0u, 0u};
  uint32_t live = 0, value = 0;
  const uint64_t g = b / ESZ;
  uint64_t row = g / ko.row_elems, ce = g - row * ko.row_elems;
  const PadDesc* d = nullptr;
#pragma unroll
  for (uint32_t j = 0; j < M; ++j) {
    if (b + (uint64_t)j * ESZ < used) {
      live |= 1u << j;
      if (!d || row < d->first_row || row >= d->first_row + d->rows) d = &pp.desc[(size_t)pad_find_rec(fr, n, row) * nk + k];
      // the element's index along every trailing axis of the destination; a value when each lies inside the record's dims
      uint64_t x = ce, lin = 0, own_stride = 1;
      bool inb = true;
      for (int32_t a = key.rank - 1; a >= 1; --a) {
        const uint64_t D = (uint64_t)key.dims[a], q = x / D, i = x - q * D;
        inb = inb && i < (uint64_t)d->dims[a];
        lin += i * own_stride;
        own_stride *= (uint64_t)d->dims[a];
        x = q;
      }
      uint64_t lo = pw[0], hi = pw[1];
      if (inb) {
        value |= 1u << j;
        if (!ko.varint) {
          const uint64_t e = (row - d->first_row) * own_stride + lin;   // own_stride is now the record's elements per row
          if (ESZ == 16) {
            lo = pad_src_bytes(*d, e * 16, 8u);
            hi = pad_src_bytes(*d, e * 16 + 8, 8u);
          } else if (ko.op == OP_F2H || ko.op == OP_F2B) {
            const uint32_t f = (uint32_t)pad_src_bytes(*d, e * 4, 4u);
            lo = ko.op == OP_F2H ? f32_bits_to_f16_bits(f) : f32_bits_to_bf16_bits(f);
          } else {
            lo = pad_src_bytes(*d, e * ESZ, ESZ);
            if (ko.op == OP_QUIET_DST) lo = quiet_f32((uint32_t)lo);
          }
        }
      }
      if (ESZ == 16) { w[0] = (uint32_t)lo; w[1] = (uint32_t)(lo >> 32); w[2] = (uint32_t)hi; w[3] = (uint32_t)(hi >> 32); }
      else if (ESZ == 8) { w[2 * j] = (uint32_t)lo; w[2 * j + 1] = (uint32_t)(lo >> 32); }
      else {
        constexpr uint64_t mask = ESZ == 4 ? 0xFFFFFFFFull : ESZ == 2 ? 0xFFFFull : 0xFFull;
        w[(j * ESZ) / 4] |= (uint32_t)(lo & mask) << (8 * ((j * ESZ) % 4));
      }
      if (++ce == ko.row_elems) { ce = 0; ++row; }
    }
  }
  uint8_t* p = key.k.dst + b;
  const uint32_t store = ko.varint ? live & ~value : live, full = (M == 32) ? ~0u : (1u << M) - 1u;
  if (store == full) { st_stream(p, make_uint4(w[0], w[1], w[2], w[3])); return; }
#pragma unroll
  for (uint32_t j = 0; j < M; ++j) {
    if (!(store >> j & 1u)) continue;
    if (ESZ == 16) *reinterpret_cast<uint4*>(p) = make_uint4(w[0], w[1], w[2], w[3]);
    else if (ESZ == 8) *reinterpret_cast<uint2*>(p + 8 * j) = make_uint2(w[2 * j], w[2 * j + 1]);
    else if (ESZ == 4) *reinterpret_cast<uint32_t*>(p + 4 * j) = w[j];
    else if (ESZ == 2) *reinterpret_cast<uint16_t*>(p + 2 * j) = (uint16_t)(w[j / 2] >> (16 * (j % 2)));
    else p[j] = (uint8_t)(w[j / 4] >> (8 * (j % 4)));
  }
}

__global__ void __launch_bounds__(kPadEmitThreads) padded_emit_kernel(const __grid_constant__ PaddedPlan pp) {
  const uint32_t nk = pp.cp.n_keys;
  const uint64_t total = pp.kout[nk].chunk0;
  for (uint64_t c = blockIdx.x; c < total; c += gridDim.x) {
    uint32_t k = 0;
    while (k + 1 < nk && pp.kout[k + 1].chunk0 <= c) ++k;
    const PadKeyOut ko = pp.kout[k];
    const PadKeyDev& key = pp.keys[k];
    const uint64_t used = ko.rows * ko.pitch;
    for (uint32_t i = 0; i < kPadEmitVecs; ++i) {
      const uint64_t b = (c - ko.chunk0) * kPadChunkBytes + 16ull * (i * kPadEmitThreads + threadIdx.x);
      if (b >= used) break;
      switch (ko.esz) {
        case 1: pad_emit_vec<1>(pp, key, ko, k, b, used); break;
        case 2: pad_emit_vec<2>(pp, key, ko, k, b, used); break;
        case 4: pad_emit_vec<4>(pp, key, ko, k, b, used); break;
        case 8: pad_emit_vec<8>(pp, key, ko, k, b, used); break;
        default: pad_emit_vec<16>(pp, key, ko, k, b, used); break;
      }
    }
  }
}

// ---- DT_STRING keys (b200tfs_decode_padded_strings; plan.h PadStrTables), behind padded_plan_strings_kernel and the emit ----
//   pad_str_index_kernel  a warp per (record, key): lane 0 walks a placed string pair's string_val elements (string_walk.h) and packs
//                         own string j's (record-relative wire offset << 32 | byte position within the pair's strings) into the
//                         offset entry of its padded position, monotone in j; the pair's own bytes go to T.bytes.  Another count
//                         than the parse's marks the pair B200TFS_E_NONCANONICAL: its rows then hold pads only.
//   pad_str_scan_kernel   one CTA: per key, a block scan of every record's bytes (own bytes + pad_len per pad position) gives its
//                         first data byte; a record past data_cap is B200TFS_E_SIZE and the rows in use end at it; offsets[m]
//                         behind them, and each key's first position among the positions to copy
//   pad_str_copy_kernel   destination-major, a lane per position: its own string (the entries of it and of the next own string
//                         give where and how long) or the pad, with warp_copy_strings; a pad position's final offset
//   pad_str_fix_kernel    the same positions: an own string's entry becomes its final offset

// entry of own string j of record d among its rows' offset entries: its index in the record's dims, mixed-radix into the
// destination's
__device__ __forceinline__ uint64_t pad_str_pos(const PadDesc& d, const PadKeyDev& key, uint64_t j) {
  uint64_t x = j, p = 0, s = 1;
  for (int32_t a = key.rank - 1; a >= 1; --a) {
    const uint64_t da = (uint64_t)d.dims[a], q = x / da;
    p += (x - q * da) * s;
    s *= (uint64_t)key.dims[a];
    x = q;
  }
  return p + x * s;
}

// StrIndexSink's placement for the padded decode, called with j = 0, 1, ...: one step along the last axis, or the whole mixed
// radix where it carries
struct PadStrPlace {
  const PadDesc* d;
  const PadKeyDev* key;
  uint64_t il, p;   // string j's index along the last axis and its entry
  __device__ __forceinline__ uint64_t operator()(uint64_t j) {
    if (j && ++il < (uint64_t)d->dims[key->rank - 1]) return ++p;
    il = 0;
    return p = pad_str_pos(*d, *key, j);
  }
};

__global__ void __launch_bounds__(kStrThreads) pad_str_index_kernel(const __grid_constant__ PadStrTables T) {
  __shared__ __align__(16) uint8_t lines[kStrThreads / 32][256];
  const ConcatPlan& cp = T.pp.cp;
  const uint32_t warp = threadIdx.x >> 5, n = cp.n, nk = cp.n_keys;
  const uint64_t q = (uint64_t)blockIdx.x * (kStrThreads / 32) + warp;   // pair r * n_keys + k
  if (q >= (uint64_t)n * nk || (threadIdx.x & 31)) return;
  const uint32_t r = (uint32_t)(q / nk), k = (uint32_t)(q % nk);
  b200tfs_output& o = cp.vouts[(size_t)r * kFusedMaxOutputs + k];
  const PadDesc& d = T.pp.desc[q];
  uint64_t total = 0;
  if (T.pp.kout[k].str && o.status == B200TFS_OK && d.rows) {
    Cursor c;
    cur_open(c, cp.w + cp.rec_off[r], (uint32_t)T.rec_len[r], lines[warp]);
    c.p = (uint32_t)o.msg_off;
    c.end = (uint32_t)(o.msg_off + o.msg_len);
    StrIndexSink<PadStrPlace> sink{reinterpret_cast<uint64_t*>((uintptr_t)o.dst_off), o.n_strings, 0u, PadStrPlace{&d, &T.pp.keys[k], 0, 0}};
    const uint64_t found = walk_strings(c, sink);
    if (c.err || found != o.n_strings) o.status = B200TFS_E_NONCANONICAL;
    else total = sink.pos;
  }
  T.bytes[(size_t)k * n + r] = total;
}

__global__ void __launch_bounds__(kConcatPlanThreads) pad_str_scan_kernel(const __grid_constant__ PadStrTables T) {
  __shared__ unsigned long long warp_sum[kConcatPlanThreads / 32];
  __shared__ unsigned long long cut_row, cut_at;   // first row and first byte of the first record past data_cap
  const PaddedPlan& pp = T.pp;
  const uint32_t n = pp.cp.n, nk = pp.cp.n_keys;
  uint64_t pos_carry = 0;
  for (uint32_t k = 0; k < nk; ++k) {
    const PadKeyOut ko = pp.kout[k];
    if (threadIdx.x == 0) T.pos0[k] = pos_carry;
    if (!ko.str) continue;                                          // uniform: every thread read the same ko
    if (threadIdx.x == 0) cut_row = cut_at = ~0ull;
    __syncthreads();
    const PadStrKeyDev sk = T.keys[k];
    uint64_t byte_carry = 0;
    for (uint32_t r0 = 0; r0 < n; r0 += kConcatPlanThreads) {      // uniform trip count: the scan has barriers inside
      const uint32_t r = r0 + threadIdx.x;
      b200tfs_output* o = nullptr;
      uint64_t pos = 0, b = 0;
      if (r < n) {
        o = &pp.cp.vouts[(size_t)r * kFusedMaxOutputs + k];
        pos = pp.desc[(size_t)r * nk + k].rows * ko.row_elems;
        const uint64_t own = o->status == B200TFS_OK ? o->n_strings : 0;   // an E_NONCANONICAL pair's rows hold pads only
        b = T.bytes[(size_t)k * n + r] + sk.pad_len * (pos - own);
      }
      const uint64_t at = concat_scan(b, byte_carry, warp_sum);
      if (r < n) {
        T.data0[(size_t)k * n + r] = at;
        if (pos && at + b > sk.cap) {
          o->status = B200TFS_E_SIZE;
          o->dst_bytes = 0;
          atomicMin(&cut_row, (unsigned long long)pp.desc[(size_t)r * nk + k].first_row);
          atomicMin(&cut_at, (unsigned long long)at);
        }
      }
    }
    __syncthreads();
    const uint64_t used = min(ko.rows, (uint64_t)cut_row), m = used * ko.row_elems;
    if (threadIdx.x == 0) {
      pp.kout[k].rows = used;
      const PadKeyDev& key = pp.keys[k];
      // offsets[m]: inside dst_cap for every record the plan placed; checked for a batch without rows
      if (8 * (m + 1) <= key.k.cap) reinterpret_cast<uint64_t*>(key.k.dst)[m] = cut_row == ~0ull ? byte_carry : (uint64_t)cut_at;
    }
    pos_carry += m;
    __syncthreads();
  }
  if (threadIdx.x == 0) T.pos0[nk] = pos_carry;
}

// position g (< T.pos0[n_keys]) of the copy and the fix: its key and record, its offset entry, whether it holds an own string, the
// own strings and the pads before it in its record's rows
struct PadStrAt {
  uint64_t* slot;        // the record's first offset entry
  uint64_t e;            // g's entry within the record's rows
  uint64_t own_before, pads_before, n_own;
  const PadDesc* d;
  uint32_t k, r;
  bool own;
};
__device__ __forceinline__ PadStrAt pad_str_at(const PadStrTables& T, uint64_t g) {
  const PaddedPlan& pp = T.pp;
  const uint32_t n = pp.cp.n, nk = pp.cp.n_keys;
  uint32_t k = 0;
  while (k + 1 < nk && T.pos0[k + 1] <= g) ++k;
  const PadKeyDev& key = pp.keys[k];
  const uint64_t re = pp.kout[k].row_elems, q = g - T.pos0[k], row = q / re, ce = q - row * re;
  PadStrAt a;
  a.k = k;
  a.r = pad_find_rec(pp.first_row + (size_t)k * n, n, row);
  a.d = &pp.desc[(size_t)a.r * nk + k];
  const b200tfs_output& o = pp.cp.vouts[(size_t)a.r * kFusedMaxOutputs + k];
  const bool ok = o.status == B200TFS_OK;
  // own tuples of the record lexicographically before the position's indices, from the last axis up; in bounds on every axis
  uint64_t x = ce, cnt = 0, own_row = 1;
  bool inb = ok;
  for (int32_t ax = key.rank - 1; ax >= 1; --ax) {
    const uint64_t D = (uint64_t)key.dims[ax], qq = x / D, i = x - qq * D, da = (uint64_t)a.d->dims[ax];
    cnt = (i < da ? cnt : 0) + min(i, da) * own_row;
    inb = inb && i < da;
    own_row *= da;
    x = qq;
  }
  const uint64_t rrow = row - a.d->first_row;
  a.slot = reinterpret_cast<uint64_t*>(key.k.dst) + a.d->first_row * re;
  a.e = rrow * re + ce;
  a.own = inb;
  a.n_own = ok ? o.n_strings : 0;
  a.own_before = ok ? rrow * own_row + cnt : 0;
  a.pads_before = a.e - a.own_before;
  return a;
}

// byte position of own string j (<= n_own) within the record's own strings
__device__ __forceinline__ uint64_t pad_str_own_pos(const PadStrTables& T, const PadStrAt& a, uint64_t j) {
  if (j == a.n_own) return T.bytes[(size_t)a.k * T.pp.cp.n + a.r];
  return (uint32_t)a.slot[pad_str_pos(*a.d, T.pp.keys[a.k], j)];
}

__global__ void __launch_bounds__(kStrThreads) pad_str_copy_kernel(const __grid_constant__ PadStrTables T) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t total = T.pos0[T.pp.cp.n_keys], step = (uint64_t)gridDim.x * kStrThreads;
#pragma unroll 1
  for (uint64_t g0 = (uint64_t)blockIdx.x * kStrThreads + (threadIdx.x & ~31u); g0 < total; g0 += step) {   // warp-uniform
    const uint64_t g = g0 + lane;
    uint8_t* dst = nullptr;
    const uint8_t* src = nullptr;
    uint64_t len = 0;
    if (g < total) {
      const PadStrAt a = pad_str_at(T, g);
      const PadStrKeyDev& sk = T.keys[a.k];
      const uint64_t base = T.data0[(size_t)a.k * T.pp.cp.n + a.r] + sk.pad_len * a.pads_before;
      if (a.own) {
        const uint64_t v = a.slot[a.e], pos = (uint32_t)v;
        src = T.pp.cp.w + T.pp.cp.rec_off[a.r] + (v >> 32);
        len = pad_str_own_pos(T, a, a.own_before + 1) - pos;
        dst = sk.data + base + pos;
      } else {
        const uint64_t at = base + pad_str_own_pos(T, a, a.own_before);
        a.slot[a.e] = at;
        src = sk.pad;
        len = sk.pad_len;
        dst = sk.data + at;
      }
    }
    warp_copy_strings(dst, src, len, g < total, UINT64_MAX);
  }
}

__global__ void __launch_bounds__(kStrThreads) pad_str_fix_kernel(const __grid_constant__ PadStrTables T) {
  const uint64_t total = T.pos0[T.pp.cp.n_keys], step = (uint64_t)gridDim.x * kStrThreads;
#pragma unroll 1
  for (uint64_t g = (uint64_t)blockIdx.x * kStrThreads + threadIdx.x; g < total; g += step) {
    const PadStrAt a = pad_str_at(T, g);
    if (a.own)
      a.slot[a.e] = T.data0[(size_t)a.k * T.pp.cp.n + a.r] + T.keys[a.k].pad_len * a.pads_before + (uint32_t)a.slot[a.e];
  }
}

cudaError_t launch_padded_strings(const PadStrTables& T, uint32_t grid, cudaStream_t stream) {
  const uint64_t pairs = (uint64_t)T.pp.cp.n * T.pp.cp.n_keys, per = kStrThreads / 32;
  pad_str_index_kernel<<<(uint32_t)((pairs + per - 1) / per), kStrThreads, 0, stream>>>(T);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  pad_str_scan_kernel<<<1, kConcatPlanThreads, 0, stream>>>(T);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  pad_str_copy_kernel<<<std::max(1u, grid), kStrThreads, 0, stream>>>(T);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  pad_str_fix_kernel<<<std::max(1u, grid), kStrThreads, 0, stream>>>(T);
  return cudaGetLastError();
}
