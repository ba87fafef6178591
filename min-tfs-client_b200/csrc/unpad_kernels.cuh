// unpad_kernels.cuh - b200tfs_encode_padded_requests_async (unpad.h): n PredictRequests cut out of one padded tensor per input,
// planned on the device.  Included by kernels.cu inside namespace b200tfs, after the move engine, the varint kernels and
// concat_scan.  Launch order, no host step between them:
//   unpad_plan_kernel    one CTA: every request's boxes from the shapes tables, rows block-scanned into first rows, statuses;
//                        the packed-varint jobs and their tile table, counters zeroed
//   unpad_len_kernel     the varint bytes of every tile (venc_len_tile over the boxes; only with a packed-varint input)
//   unpad_str_count_kernel  the string_val bytes of every string tile, and the offsets rule (only with a string input)
//   unpad_layout_kernel  one CTA: record lengths from the dims and payload lengths, a scan over the slots into rec_off, the
//                        move plan (items with their final destinations, tile table), the varint jobs' destinations, results
//   unpad_frame_kernel   one thread per request: the framing (framing.h writers through unpad_write)
//   move_kernel          the fixed-width boxes over the plan image unpad_layout_kernel wrote
//   unpad_emit_kernel    the varints (venc_emit_tile over the boxes; only with a packed-varint input)
//   unpad_str_emit_kernel   the string_val values: 42 vi(len) bytes per string (only with a string input)

// a box as the source of encode tiles (SegSrc, varint_kernels.cuh): a box that is one stretch of the padded tensor is a segment; a box
// of several runs reads each element at its padded position and goes through the same transpose
struct BoxSrc {
  UnpadIn in;
  UnpadBox b;

  __device__ __forceinline__ SegSrc seg() const { return SegSrc{in.src + b.src_off, in.src_esz, in.is_signed}; }
  __device__ __forceinline__ void load_striped(uint64_t e0, uint32_t cnt, uint64_t (&v)[kVarPerThread]) const {
    if (b.n_runs <= 1) { seg().load_striped(e0, cnt, v); return; }
    const uint8_t* base = in.src + b.src_off;
#pragma unroll
    for (uint32_t i = 0; i < kVarPerThread; ++i) {
      const uint32_t k = i * kVarThreads + threadIdx.x;
      v[i] = 0;
      if (k < cnt) {
        const uint64_t e = e0 + k, q = e / b.run;
        v[i] = ldg_elem_rt(base + (unpad_run_start(in, b, q) + (e - q * b.run)) * in.src_esz, in.src_esz, in.is_signed);
      }
    }
  }
  __device__ __forceinline__ uint32_t load_tile(uint8_t* smem, uint64_t e0, uint32_t cnt, uint64_t (&mine)[kVarPerThread], uint32_t& lens) const {
    if (b.n_runs <= 1) return seg().load_tile(smem, e0, cnt, mine, lens);
    uint64_t v[kVarPerThread];
    load_striped(e0, cnt, v);
    return venc_block_tile(smem, cnt, v, mine, lens);
  }
};

// the job of packed-varint tile t, and its box
__device__ __forceinline__ void unpad_fetch(const UnpadPlan& up, uint32_t t, VarJobDev& jb, BoxSrc& src) {
  const uint32_t s = up.tile_job[t];
  jb = up.jobs[s];
  const uint32_t r = s / up.n_var, j = up.var_in[s - r * up.n_var];
  src.in = up.ins[j];
  src.b = up.box[(size_t)r * up.F.n_in + j];
}

// kStr: the call has a string input.  A call without one runs the <false> instantiations of the plan and layout kernels, which
// compile to the code they had before string inputs existed.
template <bool kStr>
__global__ void __launch_bounds__(kConcatPlanThreads) unpad_plan_kernel(const __grid_constant__ UnpadPlan up) {
  __shared__ unsigned long long warp_sum[kConcatPlanThreads / 32];
  const uint32_t n = up.n, ni = up.F.n_in;
  uint64_t row_carry[kUnpadMaxInputs];
  for (uint32_t j = 0; j < kUnpadMaxInputs; ++j) row_carry[j] = 0;
  __shared__ unsigned long long var_cut;    // first tile of the first job past the host's bound (never with it)
  if (threadIdx.x == 0) var_cut = ~0ull;
  if (kStr && threadIdx.x == 0) *up.n_str_tiles = up.str_tile_cap;   // lowered like var_cut, then to the tiles planned
  __syncthreads();
  uint64_t tile_carry = 0, group_carry = 0, str_tile_carry = 0, str_group_carry = 0;
  for (uint32_t r0 = 0; r0 < n; r0 += kConcatPlanThreads) {       // uniform trip counts: the scans have barriers inside
    const uint32_t r = r0 + threadIdx.x;
    const bool live = r < n;
    int32_t st = B200TFS_OK;
    for (uint32_t j = 0; j < ni; ++j) {
      const UnpadIn& in = up.ins[j];
      UnpadBox b{};
      int32_t s = B200TFS_OK;
      if (live) s = unpad_box(in, in.shapes ? in.shapes + (size_t)r * in.cols : nullptr, &b);
      if (in.shapes) {
        const uint64_t rows = live ? (uint64_t)b.dims[0] : 0;   // a bad trailing dim keeps its rows: the requests behind it stay put
        const uint64_t first = concat_scan(rows, row_carry[j], warp_sum);
        if (live && s == B200TFS_OK && first + rows > (uint64_t)in.dims[0]) s = B200TFS_E_SIZE;
        uint64_t pitch = in.src_esz;
        for (int32_t d = 1; d < in.rank; ++d) pitch *= (uint64_t)in.dims[d];
        b.src_off = first * pitch;
      }
      if (live) {
        if (st == B200TFS_OK) st = s;
        up.box[(size_t)r * ni + j] = b;
      }
    }
    if (live) up.st[r] = st;
    for (uint32_t v = 0; v < up.n_var; ++v) {
      const uint32_t j = up.var_in[v];
      const uint64_t ne = (live && st == B200TFS_OK) ? up.box[(size_t)r * ni + j].n_elems : 0;
      const uint64_t tiles = (ne + kVarTileElems - 1) / kVarTileElems, groups = (tiles + kVarGroupTiles - 1) / kVarGroupTiles;
      const uint64_t first = concat_scan(tiles, tile_carry, warp_sum);
      const uint64_t group0 = concat_scan(groups, group_carry, warp_sum);   // every job's counter groups apart from all others
      // past the bound (never: unpad_bounds): tiles only grow in scan order, so such jobs are a suffix - their requests get
      // B200TFS_E_SIZE, and the tile count stops at the first one
      const bool over = first + tiles > up.var_tile_cap || group0 + groups > up.var_group_cap;
      if (over) atomicMin(&var_cut, (unsigned long long)first);
      if (live) {
        const uint64_t s = (uint64_t)r * up.n_var + v;
        if (over) { st = B200TFS_E_SIZE; up.st[r] = st; }
        const UnpadIn& in = up.ins[j];
        VarJobDev jb{};
        jb.dst = up.arena;                       // parked until unpad_layout_kernel places the record
        jb.n_elems = over ? 0 : ne;
        jb.tile_val = up.tile_val + first;
        jb.group_sum = up.group_sum + group0;
        jb.total = up.total + s;
        jb.dtype = in.wire_dtype;
        jb.elem_size = in.src_esz;
        jb.is_signed = in.is_signed;
        jb.first_tile = (uint32_t)first;
        jb.n_tiles = (uint32_t)tiles;
        if (!over) {
          for (uint64_t i = 0; i < tiles; ++i) up.tile_job[first + i] = (uint32_t)s;
          for (uint64_t g = 0; g < groups; ++g) jb.group_sum[g] = 0;
        }
        *jb.total = 0;
        up.jobs[s] = jb;
      }
    }
    // string jobs: every good box gets a tile, an empty one too (unpad_str_count_kernel checks its outer offsets there)
    for (uint32_t k = 0; kStr && k < up.n_str; ++k) {
      const uint32_t j = up.str_in[k];
      const bool ok = live && st == B200TFS_OK;
      const uint64_t ne = ok ? up.box[(size_t)r * ni + j].n_elems : 0;
      const uint64_t tiles = ok ? max((ne + kVarThreads - 1) / kVarThreads, (uint64_t)1) : 0, groups = (tiles + kVarGroupTiles - 1) / kVarGroupTiles;
      const uint64_t first = concat_scan(tiles, str_tile_carry, warp_sum);
      const uint64_t group0 = concat_scan(groups, str_group_carry, warp_sum);
      const bool over = first + tiles > up.str_tile_cap || group0 + groups > up.str_group_cap;   // never: unpad_bounds
      if (over) atomicMin(up.n_str_tiles, (uint32_t)min(first, (uint64_t)up.str_tile_cap));
      if (live) {
        const uint64_t s = (uint64_t)r * up.n_str + k;
        if (over) { st = B200TFS_E_SIZE; up.st[r] = st; }
        VarJobDev jb{};
        jb.dst = up.arena;
        jb.n_elems = over ? 0 : ne;
        jb.tile_val = up.str_tile_val + first;
        jb.group_sum = up.str_group_sum + group0;
        jb.total = up.str_total + s;
        jb.first_tile = (uint32_t)first;
        jb.n_tiles = over ? 0 : (uint32_t)tiles;
        if (!over) {
          for (uint64_t i = 0; i < tiles; ++i) up.str_tile_job[first + i] = (uint32_t)s;
          for (uint64_t g = 0; g < groups; ++g) jb.group_sum[g] = 0;
        }
        *jb.total = 0;
        up.str_jobs[s] = jb;
      }
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) *up.n_var_tiles = (uint32_t)min(min(tile_carry, (uint64_t)var_cut), (uint64_t)up.var_tile_cap);
  if (kStr && threadIdx.x == 0) atomicMin(up.n_str_tiles, (uint32_t)min(str_tile_carry, (uint64_t)up.str_tile_cap));
}

__global__ void __launch_bounds__(kVarThreads) unpad_len_kernel(const __grid_constant__ UnpadPlan up) {
  __shared__ VarShared sh;
  const uint32_t t = blockIdx.x;
  if (t >= *up.n_var_tiles) return;
  VarJobDev jb;
  BoxSrc src;
  unpad_fetch(up, t, jb, src);
  const uint32_t t_rel = t - jb.first_tile;
  const uint64_t e0 = (uint64_t)t_rel * kVarTileElems;
  venc_len_tile(sh, jb, t_rel, e0, (uint32_t)min((uint64_t)kVarTileElems, jb.n_elems - e0), src);
}

// fixed-width moves of one (request, input): one item for a box that is one stretch of the source (the engine's vector path), else
// one gathered item per index of the axes above lo - 1, each a row of dims[lo - 1] pieces of `run` elements
struct UnpadItems { uint64_t items, per_item_runs, item_bytes; uint32_t tiles_per_item; };
template <bool kStr>
__device__ __forceinline__ UnpadItems unpad_items(const UnpadIn& in, const UnpadBox& b, uint32_t vpt) {
  UnpadItems I{0, 0, 0, 0};
  if (in.varint || (kStr && in.str) || !b.n_elems) return I;
  I.per_item_runs = b.n_runs <= 1 ? 1 : (uint64_t)b.dims[b.lo - 1];
  I.items = b.n_runs <= 1 ? 1 : b.n_runs / I.per_item_runs;
  I.item_bytes = I.per_item_runs * b.run * in.wire_esz;
  I.tiles_per_item = tiles_for(I.item_bytes, vpt);
  return I;
}

template <bool kStr>
__global__ void __launch_bounds__(kConcatPlanThreads) unpad_layout_kernel(const __grid_constant__ UnpadPlan up) {
  __shared__ unsigned long long warp_sum[kConcatPlanThreads / 32];
  const uint32_t n = up.n, ni = up.F.n_in;
  const PlanGeometry g = plan_geometry(up.item_cap, up.tile_cap, 0);
  MoveItem* items = reinterpret_cast<MoveItem*>(up.plan + g.off_items);
  TileRef* tref = reinterpret_cast<TileRef*>(up.plan + g.off_tiles);
  __shared__ unsigned long long tile_cut;   // first tile of the first request past the host's bounds (never with them)
  if (threadIdx.x == 0) tile_cut = ~0ull;
  __syncthreads();
  uint64_t slot_carry = 0, item_carry = 0, tile_carry = 0;
  for (uint32_t r0 = 0; r0 < n; r0 += kConcatPlanThreads) {
    const uint32_t r = r0 + threadIdx.x;
    const bool live = r < n;
    int32_t st = live ? up.st[r] : B200TFS_E_ARG;
    UnpadBox* B = up.box + (size_t)r * ni;
    uint64_t poff[kUnpadMaxInputs];
    uint64_t len = 0, largest_off = 0, n_items = 0, n_tiles = 0;
    if (st == B200TFS_OK) {
      for (uint32_t j = 0, v = 0, k = 0; j < ni; ++j) {
        const UnpadIn& in = up.ins[j];
        const uint64_t ne = B[j].n_elems;
        B[j].payload = in.varint ? (ne ? (uint64_t)up.total[(size_t)r * up.n_var + v] : 0)
                     : kStr && in.str ? (ne ? (uint64_t)up.str_total[(size_t)r * up.n_str + k] : 0) : ne * in.wire_esz;
        v += in.varint;
        if (kStr) k += in.str != 0;
      }
      int32_t s2;
      len = unpad_layout(up.F, up.ins, B, poff, &largest_off, &s2);
      st = s2;
    }
    const uint64_t pad = (128 - (largest_off & 127)) & 127;
    const uint64_t slot = st == B200TFS_OK ? (pad + len + 255) & ~255ull : 0;
    const uint64_t at = concat_scan(slot, slot_carry, warp_sum);
    if (st == B200TFS_OK && at + pad + len > up.arena_cap) st = B200TFS_E_SIZE;   // never with b200tfs_padded_request_arena_size bytes
    if (st == B200TFS_OK)
      for (uint32_t j = 0; j < ni; ++j) {
        const UnpadItems I = unpad_items<kStr>(up.ins[j], B[j], up.vpt);
        n_items += I.items;
        n_tiles += I.items * I.tiles_per_item;
      }
    const uint64_t first_item = concat_scan(n_items, item_carry, warp_sum);
    const uint64_t first_tile = concat_scan(n_tiles, tile_carry, warp_sum);
    if (!live) continue;
    // Past the host's bounds (never: unpad_bounds).  Item and tile starts only grow, so the requests past them are a suffix: they get
    // B200TFS_E_SIZE and no moves, and the plan stops at the first one's tiles - every tile in front of it has its reference written.
    if (first_item + n_items > up.item_cap || first_tile + n_tiles > up.tile_cap) {
      st = B200TFS_E_SIZE;
      atomicMin(&tile_cut, (unsigned long long)first_tile);
    }
    const uint64_t rec = at + pad;
    if (st == B200TFS_OK) {
      uint64_t it = first_item, tt = first_tile;
      for (uint32_t j = 0, v = 0, k = 0; j < ni; ++j) {
        const UnpadIn& in = up.ins[j];
        const UnpadBox& b = B[j];
        uint8_t* dst = up.arena + rec + poff[j];
        if (kStr && in.str) {
          VarJobDev& jb = up.str_jobs[(size_t)r * up.n_str + k];
          jb.dst = dst; jb.cap = b.payload;
          ++k;
          continue;
        }
        if (in.varint) {
          VarJobDev& jb = up.jobs[(size_t)r * up.n_var + v];
          jb.dst = dst; jb.cap = b.payload;
          ++v;
          continue;
        }
        const UnpadItems I = unpad_items<kStr>(in, b, up.vpt);
        uint64_t pitch = in.src_esz;      // source bytes of one index of axis lo - 1
        for (int32_t d = (int32_t)b.lo; d < in.rank; ++d) pitch *= (uint64_t)in.dims[d];
        for (uint64_t k = 0; k < I.items; ++k, ++it) {
          const uint8_t* src = in.src + b.src_off + unpad_run_start(in, b, k * I.per_item_runs) * in.src_esz;
          const bool gather = b.n_runs > 1;
          items[it] = MoveItem{src, dst + k * I.item_bytes, I.item_bytes, in.op, I.tiles_per_item,
                               gather ? (uint32_t)(b.run * in.src_esz) : 0u, gather ? (uint32_t)pitch : 0u};
          for (uint32_t q = 0; q < I.tiles_per_item; ++q) tref[tt++] = TileRef{(uint32_t)it, q};
        }
      }
    } else {
      for (uint32_t v = 0; v < up.n_var; ++v) { VarJobDev& jb = up.jobs[(size_t)r * up.n_var + v]; jb.dst = up.arena; jb.cap = 0; }
      for (uint32_t k = 0; kStr && k < up.n_str; ++k) { VarJobDev& jb = up.str_jobs[(size_t)r * up.n_str + k]; jb.dst = up.arena; jb.cap = 0; }
    }
    up.st[r] = st;
    up.rec_off[r] = st == B200TFS_OK ? rec : 0;
    up.rec_off[n + r] = st == B200TFS_OK ? len : 0;
    up.rec_off_host[r] = st == B200TFS_OK ? rec : 0;
    up.rec_len_host[r] = st == B200TFS_OK ? len : 0;
    up.status_host[r] = st;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    PlanHeader ph{};
    ph.n_items = up.item_cap;
    ph.n_tiles = (uint32_t)min(min(tile_carry, (uint64_t)tile_cut), (uint64_t)up.tile_cap);
    ph.vec_per_tile = up.vpt;
    ph.off_items = (uint32_t)g.off_items;
    ph.off_tiles = (uint32_t)g.off_tiles;
    ph.off_small = (uint32_t)g.off_small;
    ph.guard_div = 1;
    *reinterpret_cast<PlanHeader*>(up.plan) = ph;
  }
}

__global__ void __launch_bounds__(kUnpadFrameThreads) unpad_frame_kernel(const __grid_constant__ UnpadPlan up) {
  const uint32_t r = blockIdx.x * kUnpadFrameThreads + threadIdx.x;
  if (r >= up.n || up.st[r] != B200TFS_OK) return;
  RawOut o{up.arena + up.rec_off[r]};
  unpad_write(o, up.F, up.ins, up.box + (size_t)r * up.F.n_in, up.rec_off[up.n + r] - (up.F.grpc ? 5 : 0), nullptr);
}

__global__ void __launch_bounds__(kVarThreads, 5) unpad_emit_kernel(const __grid_constant__ UnpadPlan up) {
  __shared__ __align__(16) uint8_t smem[kVarImageBytes];
  __shared__ VarShared sh;
  const uint32_t t = blockIdx.x;
  if (t >= *up.n_var_tiles) return;
  VarJobDev jb;
  BoxSrc src;
  unpad_fetch(up, t, jb, src);
  const uint32_t t_rel = t - jb.first_tile;
  const uint64_t e0 = (uint64_t)t_rel * kVarTileElems;
  venc_emit_tile(smem, sh, jb, t_rel, e0, (uint32_t)min((uint64_t)kVarTileElems, jb.n_elems - e0), src);
}

// ---- string columns (unpad.h "string columns") --------------------------------------------------------------------------------
// A string tile is kVarThreads strings of one job, a thread per string; its wire bytes go into the job's tables as a varint
// tile's do (publish_tile), so the emit finds a tile's first byte with prefix_share.

// the job of string tile t, its box and the tile's first string; false: nothing to do (past the tiles planned, a bad request)
__device__ __forceinline__ bool unpad_str_fetch(const UnpadPlan& up, uint32_t t, VarJobDev& jb, UnpadIn& in, UnpadStrCol& col,
                                                UnpadBox& b, uint32_t& r) {
  if (t >= *up.n_str_tiles) return false;
  const uint32_t s = up.str_tile_job[t];
  r = s / up.n_str;
  if (up.st[r] != B200TFS_OK) return false;
  jb = up.str_jobs[s];
  const uint32_t k = s - r * up.n_str, j = up.str_in[k];
  in = up.ins[j];
  col = up.str_cols[k];
  b = up.box[(size_t)r * up.F.n_in + j];
  return true;
}

// string e of the box (e < n_elems): its clamped start and length; *ok drops if an offset is out of range or the end is before
// the start
__device__ __forceinline__ uint64_t unpad_str_span(const UnpadIn& in, const UnpadStrCol& col, const UnpadBox& b, uint64_t e,
                                                   uint64_t* start, bool* ok) {
  const uint64_t i = unpad_str_index(in, b, e);
  const uint64_t s0 = unpad_str_off(col, i, ok), s1 = unpad_str_off(col, i + 1, ok);
  if (s1 < s0) *ok = false;
  *start = s0;
  return s1 > s0 ? s1 - s0 : 0;
}

__global__ void __launch_bounds__(kVarThreads) unpad_str_count_kernel(const __grid_constant__ UnpadPlan up) {
  __shared__ VarShared sh;
  VarJobDev jb;
  UnpadIn in;
  UnpadStrCol col;
  UnpadBox b;
  uint32_t r;
  if (!unpad_str_fetch(up, blockIdx.x, jb, in, col, b, r)) return;
  const uint32_t t_rel = blockIdx.x - jb.first_tile;
  const uint64_t e = (uint64_t)t_rel * kVarThreads + threadIdx.x;
  uint64_t first, end;
  unpad_str_rows(in, b, &first, &end);
  bool ok = true;
  uint64_t size = 0;
  if (e < jb.n_elems) {   // the offsets rule around string e: what is read before its start, its end, and after the last one
    uint64_t s0;
    const uint64_t len = unpad_str_span(in, col, b, e, &s0, &ok);
    const uint64_t before = unpad_str_off(col, e ? unpad_str_index(in, b, e - 1) + 1 : first, &ok);
    if (before > s0) ok = false;
    if (e + 1 == jb.n_elems && s0 + len > unpad_str_off(col, end, &ok)) ok = false;
    size = string_value_len(len);
  }
  if (t_rel == 0 && threadIdx.x == 0 && unpad_str_off(col, first, &ok) > unpad_str_off(col, end, &ok)) ok = false;   // empty boxes too
  uint32_t unused;
  uint64_t total;
  block_scan_sum(0, &unused, size, &total, sh);
  const bool bad = __syncthreads_or(!ok);
  if (threadIdx.x == 0) {
    if (bad) up.st[r] = B200TFS_E_SHAPE;
    publish_tile(jb, t_rel, (uint32_t)min(total, (uint64_t)0xFFFFFFFFu));   // a saturated tile makes the request too big
  }
}

// Strings up to kStrLaneCopy bytes are copied by their own thread, up to kUnpadStrBlockCopy by their warp, longer ones by the CTA.
constexpr uint64_t kUnpadStrBlockCopy = 16384;

__global__ void __launch_bounds__(kVarThreads) unpad_str_emit_kernel(const __grid_constant__ UnpadPlan up) {
  __shared__ VarShared sh;
  __shared__ uint32_t n_long;
  __shared__ uint64_t long_src[kVarThreads], long_dst[kVarThreads], long_len[kVarThreads];
  VarJobDev jb;
  UnpadIn in;
  UnpadStrCol col;
  UnpadBox b;
  uint32_t r;
  if (!unpad_str_fetch(up, blockIdx.x, jb, in, col, b, r)) return;   // the layout kernel's final statuses: a bad request writes nothing
  if (threadIdx.x == 0) n_long = 0;
  const uint32_t t_rel = blockIdx.x - jb.first_tile;
  const uint64_t e = (uint64_t)t_rel * kVarThreads + threadIdx.x;
  bool ok = true;
  uint64_t s0 = 0, len = 0, size = 0;
  if (e < jb.n_elems) {
    len = unpad_str_span(in, col, b, e, &s0, &ok);   // the lengths the count read
    size = string_value_len(len);
  }
  uint32_t tile_total;
  uint64_t base;
  const uint32_t pos = block_scan_sum((uint32_t)size, &tile_total, prefix_share(jb, t_rel), &base, sh);   // (barriers inside)
  uint8_t* d = jb.dst + base + pos;
  const bool mine = size && base + pos + size <= jb.cap;   // always, for a request that counted its bytes
  if (mine) {
    RawOut o{d};
    o.byte(0x42);
    o.varint(len);
    d = o.w;
  }
  warp_copy_strings(d, in.src + s0, len, mine, kUnpadStrBlockCopy);
  if (mine && len > kUnpadStrBlockCopy) {
    const uint32_t q = atomicAdd(&n_long, 1u);
    long_src[q] = s0; long_dst[q] = (uint64_t)(uintptr_t)d; long_len[q] = len;
  }
  __syncthreads();
#pragma unroll 1
  for (uint32_t q = 0; q < n_long; ++q)
    copy_bytes((uint8_t*)(uintptr_t)long_dst[q], in.src + long_src[q], long_len[q], threadIdx.x, kVarThreads);
}

cudaError_t launch_unpad(const UnpadPlan& up, uint32_t move_grid, cudaStream_t stream, uint32_t* launched) {
  *launched = 0;
  if (!up.n) return cudaSuccess;
  const uint32_t var_grid = up.n_var ? up.var_tile_cap : 0;
  const uint32_t str_grid = up.n_str ? up.str_tile_cap : 0;
  if (str_grid) unpad_plan_kernel<true><<<1, kConcatPlanThreads, 0, stream>>>(up);
  else unpad_plan_kernel<false><<<1, kConcatPlanThreads, 0, stream>>>(up);
  ++*launched;
  if (var_grid) { unpad_len_kernel<<<var_grid, kVarThreads, 0, stream>>>(up); ++*launched; }
  if (str_grid) { unpad_str_count_kernel<<<str_grid, kVarThreads, 0, stream>>>(up); ++*launched; }
  if (str_grid) unpad_layout_kernel<true><<<1, kConcatPlanThreads, 0, stream>>>(up);
  else unpad_layout_kernel<false><<<1, kConcatPlanThreads, 0, stream>>>(up);
  unpad_frame_kernel<<<(up.n + kUnpadFrameThreads - 1) / kUnpadFrameThreads, kUnpadFrameThreads, 0, stream>>>(up);
  *launched += 2;
  // a plain launch, as in launch_concat_plan: the kernel in front of move_kernel writes its plan header
  if (move_grid) { move_kernel<<<move_grid, kMoveThreads, 0, stream>>>((const uint8_t*)up.plan); ++*launched; }
  if (var_grid) { unpad_emit_kernel<<<var_grid, kVarThreads, 0, stream>>>(up); ++*launched; }
  if (str_grid) { unpad_str_emit_kernel<<<str_grid, kVarThreads, 0, stream>>>(up); ++*launched; }
  return cudaGetLastError();
}
