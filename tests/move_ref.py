"""Reference of the fixed-width move engine (csrc/kernels.cu: move_tile, its vector bodies, the byte generator and the staged
tile of the batch decode): the bytes each op writes, and a model of the engine's geometry - which body a tile takes, how many
vectors and rounds it moves, and every 16-byte block it loads - computed from the real source and destination addresses.

The GPU edge tests (tests/test_move_edges_gpu.py) compare the device with the byte references and use the geometry model to
assert which edges they reached; tests/test_move_reference_cpu.py pins both.  The engine's constants are read from the sources,
so the model cannot drift silently from the kernels.
"""
import os
import re

import numpy as np

from oracle import wire_oracle

_CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "min-tfs-client_b200", "csrc")


def _const(fname, name):
    with open(os.path.join(_CSRC, fname)) as f:
        m = re.search(r"constexpr\s+uint32_t\s+%s\s*=\s*(\d+)u?\s*;" % name, f.read())
    assert m, (fname, name)
    return int(m.group(1))


K_SMALL_MAX = _const("plan.h", "kSmallMax")              # payloads up to this many bytes: one warp (SmallItem)
K_MOVE_THREADS = _const("plan.h", "kMoveThreads")
K_INLINE_PLAN_BYTES = _const("plan.h", "kInlinePlanBytes")
K_STAGE_VECS = _const("kernels.h", "kStageVecsHost")      # destination vectors per staged chunk
K_BATCH_ALIGNED = _const("kernels.cu", "kBatchAligned")
K_BATCH_SHIFT = _const("kernels.cu", "kBatchShift")
K_STAGE_BUFS = _const("kernels.cu", "kStageBufs")

ROUND_ALIGNED = K_BATCH_ALIGNED * K_MOVE_THREADS          # vectors per round of body_aligned
ROUND_SHIFT = K_BATCH_SHIFT * K_MOVE_THREADS              # body_shifted_q: kBatchShift * 32 per warp, 8 warps
ROUND_NARROW = 4 * K_MOVE_THREADS                         # body_narrow_q: kU = 4 output vectors per lane
ROUND_WIDEN = 8 * K_MOVE_THREADS                          # body_widen: 8 units per thread

COPY, QUIET_SRC, QUIET_DST, BOOL, H2F, B2F, F2H, F2B = range(8)
OPS = {"COPY": COPY, "QUIET_SRC": QUIET_SRC, "QUIET_DST": QUIET_DST, "BOOL": BOOL, "H2F": H2F, "B2F": B2F, "F2H": F2H, "F2B": F2B}


# ---- the bytes each op writes -----------------------------------------------------------------------------------------------
def quiet_f32(bits):
    """float32 NaNs with the quiet bit set (w | 0x00400000), every other pattern unchanged."""
    w = np.asarray(bits).view(np.uint32)
    return np.where((w & 0x7FFFFFFF) > 0x7F800000, w | np.uint32(0x00400000), w).astype(np.uint32)


def gather(src, glen, gstride, n):
    """The logical source stream of a run of unpacked elements: byte j lies at src[(j // glen) * gstride + j % glen]."""
    src = np.frombuffer(bytes(src), np.uint8)
    j = np.arange(n, dtype=np.int64)
    return src[(j // glen) * gstride + j % glen]


def out_bytes(op, src):
    """The bytes `op` writes for a whole source stream `src` (bytes-like): what the byte generator and every vector body
    must produce."""
    s = np.frombuffer(bytes(src), np.uint8)
    if op == COPY:
        return s.tobytes()
    if op == BOOL:
        return (s != 0).astype(np.uint8).tobytes()
    if op in (QUIET_SRC, QUIET_DST):
        return quiet_f32(s.view(np.uint32)).tobytes()
    if op in (H2F, B2F):
        import ml_dtypes
        return wire_oracle.widen_16(s.view(np.float16 if op == H2F else ml_dtypes.bfloat16)).tobytes()
    if op in (F2H, F2B):
        import ml_dtypes
        return wire_oracle.narrow_f32(s.view(np.float32), np.float16 if op == F2H else ml_dtypes.bfloat16).tobytes()
    raise ValueError(op)


def src_bytes_for(op, n_out):
    if op in (H2F, B2F):
        return n_out >> 1
    if op in (F2H, F2B):
        return n_out << 1
    return n_out


# ---- geometry ---------------------------------------------------------------------------------------------------------------
def tiles_for(n_out, vpt):
    vecs = (n_out + 15) >> 4
    return max(1, (vecs + vpt - 1) // vpt)


def pick_vec_per_tile(sm_count, large_bytes, max_tile, override=0):
    """codec_host.cpp pick_vec_per_tile: about 8 tiles per SM in whole 32 KB, capped at max_tile (32 KB for an encode or
    unpack plan, 64 KB for the batch decode); B200TFS_TILE_BYTES overrides it."""
    tile = override
    if not tile:
        target = sm_count * 8
        tile = (large_bytes + target - 1) // target
        tile = (tile + 32767) & ~32767
        tile = min(max(tile, 32768), max_tile)
    tile = max(tile & ~31, 32)
    return tile // 16


class Geometry:
    """What move_tile<DEC> does with one payload: src / dst are the real addresses of the payload's first source and
    destination bytes."""

    def __init__(self, src, dst, n_out, op, dec=False):
        self.src, self.dst, self.n_out, self.op, self.dec = src, dst, n_out, op, dec
        self.n_src = n_out if dec else src_bytes_for(op, n_out)
        head = min((16 - (dst & 15)) & 15, n_out)
        fast = True
        if dec or op in (COPY, QUIET_SRC, QUIET_DST, BOOL):
            self.kind = "same"
            if not dec and op == QUIET_SRC:
                fast = (src & 3) == 0
            if op == QUIET_DST:
                fast = (head & 3) == 0
            nvec = (n_out - head) >> 4
            body = src + head
            k = body & 15
            if k:
                blocks = ((src + self.n_src) - (body - k)) >> 4
                nvec = min(nvec, blocks - 1 if blocks else 0)
        elif op in (H2F, B2F):
            self.kind = "widen"
            body = src
            fast = head == 0 and (src & 15) == 0
            nvec = (n_out >> 5) << 1
            k = src & 15
        else:
            self.kind = "narrow"
            body = src + 2 * head
            fast = (head & 1) == 0
            nvec = (n_out - head) >> 4
            k = body & 15
            span = (src + self.n_src) - (body - k)
            lim = ((span - 16) >> 5 if span >= 16 else 0) if k else span >> 5
            nvec = min(nvec, lim)
        self.head, self.fast, self.nvec, self.k, self.src_body = head, fast, nvec, k, body
        self.tail = n_out - head - 16 * nvec if fast else 0

    @property
    def dphase(self):
        return self.dst & 15

    def body(self):
        """Vector body the tiles take (None: the byte generator for the whole payload)."""
        if not self.fast:
            return None
        if self.kind == "same":
            return "aligned" if self.k == 0 else "shifted%d" % (self.k >> 2)
        if self.kind == "widen":
            return "widen"
        return "narrow" if self.k == 0 else "narrow%d" % (self.k >> 2)

    def round_vecs(self):
        b = self.body()
        if b == "aligned":
            return ROUND_ALIGNED
        if b and b.startswith("shifted"):
            return ROUND_SHIFT
        if b == "widen":
            return 2 * ROUND_WIDEN
        return ROUND_NARROW

    def tiles(self, vpt):
        """[(tile, first vector, vectors, rounds of its body)] of a tiled payload."""
        out = []
        for t in range(tiles_for(self.n_out, vpt)):
            v0 = t * vpt
            n = min(vpt, self.nvec - v0) if self.fast and v0 < self.nvec else 0
            out.append((t, v0, n, -(-n // self.round_vecs()) if n else 0))
        return out

    def writes(self, vpt):
        """[(tile, start, end)] destination byte ranges of every tile, head and tail included (payload-relative)."""
        w = []
        nt = tiles_for(self.n_out, vpt)
        if not self.fast:
            for t in range(nt):
                b0 = t * vpt * 16
                b1 = self.n_out if (t + 1 == nt or b0 + vpt * 16 > self.n_out) else b0 + vpt * 16
                if b1 > b0:
                    w.append((t, b0, b1))
            return w
        for t, v0, n, _ in self.tiles(vpt):
            if t == 0 and self.head:
                w.append((t, 0, self.head))
            if n:
                w.append((t, self.head + 16 * v0, self.head + 16 * (v0 + n)))
            if t + 1 == nt and self.head + 16 * self.nvec < self.n_out:
                w.append((t, self.head + 16 * self.nvec, self.n_out))
        return w

    def loads(self, vpt):
        """[(start, end)] absolute source byte ranges the vector bodies load (128-bit loads: the byte generator's exact reads
        are left out)."""
        out = []
        if not self.fast:
            return out
        S = self.src_body - self.k
        for t, v0, n, _ in self.tiles(vpt):
            if not n:
                continue
            if self.kind == "same":
                # blocks v of the tile, and (shifted) block v+1 of its last vector: the run's `extra`
                out.append((S + 16 * v0, S + 16 * (v0 + n + (1 if self.k else 0))))
            elif self.kind == "widen":
                out.append((self.src_body + 8 * v0, self.src_body + 8 * v0 + 16 * (n >> 1)))
            else:
                out.append((S + 32 * v0, S + 32 * (v0 + n) + (16 if self.k else 0)))
        return out

    def staged(self, vpt):
        """staged_begin for the fused batch decode (dec): None when the geometry does not qualify (move_tile_cold), else
        [(tile, [(chunk, vectors, bulk bytes, source offset from S, parity of its wait)])]."""
        if self.op not in (COPY, QUIET_DST) or (self.op == QUIET_DST and (self.head & 3)):
            return None
        out = []
        for t, v0, n, _ in self.tiles(vpt):
            chunks = []
            for c in range(-(-n // K_STAGE_VECS)):
                nc = min(K_STAGE_VECS, n - c * K_STAGE_VECS)
                chunks.append((c, nc, 16 * (nc + (1 if self.k else 0)), 16 * (v0 + c * K_STAGE_VECS), (c // K_STAGE_BUFS) & 1))
            out.append((t, chunks))
        return out

    def read_window(self):
        """[floor16(src), ceil16(src + n_src)): every load must stay inside (a load there cannot fault)."""
        return self.src & ~15, (self.src + self.n_src + 15) & ~15


def route(n_out):
    """Encode and unpack plans give payloads of up to kSmallMax bytes to one warp (the fused decode tiles every payload)."""
    return "warp" if n_out <= K_SMALL_MAX else "tile"


# plan.h: sizeof(PlanHeader) / MoveItem / TileRef / SmallItem on a 64-bit host (pinned against the struct definitions by
# tests/test_move_reference_cpu.py)
PLAN_HEADER_BYTES, MOVE_ITEM_BYTES, TILE_REF_BYTES, SMALL_ITEM_BYTES = 56, 40, 8, 32


def plan_image(n_items, n_tile_refs, n_small, blob):
    """Bytes of a plan image (plan_geometry, then the header blob): at most kInlinePlanBytes travel in the kernel parameters
    (move_kernel_inline), larger images are uploaded (move_kernel)."""
    off_items = (PLAN_HEADER_BYTES + 15) & ~15
    off_tiles = off_items + n_items * MOVE_ITEM_BYTES
    off_small = (off_tiles + n_tile_refs * TILE_REF_BYTES + 15) & ~15
    return off_small + n_small * SMALL_ITEM_BYTES + blob


def inline_plan(image):
    return image <= K_INLINE_PLAN_BYTES
