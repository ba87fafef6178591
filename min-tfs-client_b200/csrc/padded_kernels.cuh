// padded_kernels.cuh - b200tfs_decode_padded: a batch of PredictResponses into one padded tensor per requested key (plan.h
// PaddedPlan; the host side is in codec_host.cpp).  Included by kernels.cu inside namespace b200tfs, after concat_plan_kernel.
//
//   padded_plan_kernel  one CTA.  Per key: concat_plan_kernel's pass A (plan_key_reference), then every record against the first
//                       record that decoded the key (dtype, rank) and against the destination's trailing dims, a block scan of
//                       dims[0] into first rows, one PadDesc per (record, key) and the single-launch decode's table for the
//                       varint tail.  Nothing waits on another CTA: a replayed graph re-plans rows and trailing dims.
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

__global__ void __launch_bounds__(kConcatPlanThreads) padded_plan_kernel(const __grid_constant__ PaddedPlan pp) {
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
    const uint32_t esz = narrow ? 2u : di.elem_size;
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
          // strings are decoded on the host; the emit reads the inline runs only; the varint decode takes packed occurrences only
          if (kind == VK_STRING || (o->flags & B200TFS_OF_SPILLED) || o->n_inline != (uint32_t)o->n_runs) st = B200TFS_E_NONCANONICAL;
          if (kind == VK_VARINT || kind == VK_BOOL) {
            if (o->flags & B200TFS_OF_UNPACKED) st = B200TFS_E_NONCANONICAL;
            for (int32_t q = 0; q < o->n_runs && q < B200TFS_MAX_RUNS; ++q) if (o->runs[q].count != 1) st = B200TFS_E_NONCANONICAL;
          }
        }
        if (st == B200TFS_OK) rows = (uint64_t)o->dims[0];
      }
      const uint64_t first = concat_scan(rows, row_carry, warp_sum);
      if (r < n) {
        if (st == B200TFS_OK && rows && (first + rows) * pitch > key.k.cap) {
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
      pp.kout[k] = ko;
      chunks += (used * pitch + kPadChunkBytes - 1) / kPadChunkBytes;
    }
  }
  if (threadIdx.x == 0) { PadKeyOut end{}; end.chunk0 = chunks; pp.kout[nk] = end; }
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
