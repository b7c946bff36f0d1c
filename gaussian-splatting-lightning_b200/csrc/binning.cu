// K2-K5: tile binning.
//
// The reference backends sort I (tile,Gaussian) pairs on a 64-bit (tile | depth-bits) key: ~6 radix passes over
// 12 B pairs (SURVEY §8d: I*152 B, the largest pure-bandwidth term of their forward).  The same total order — tile
// major, then depth bits, ties in Gaussian-id order — is produced here hierarchically, and the fine pairs are written
// exactly once, already in place:
//   A. depth keys (32-bit float bits; off-screen -> 0xFFFFFFFF), stable radix sort of the N keys, scan of the
//      per-Gaussian COARSE cell counts in depth order (a coarse cell = 8x8 tiles = 128x128 px); a 32-byte record per
//      Gaussian (one L2 sector) holds everything phase B needs
//   B. emit (coarse cell, {64-bit tile mask, id}) pairs in depth order — the mask = which of the cell's 64 tiles the splat
//      can reach (row spans of the alpha >= 1/255 ellipse, or the plain 3-sigma rect with culling off) — and
//      stable-partition them by cell: ONE 8-bit radix pass over ~2 pairs per visible Gaussian for every image up to
//      2048x2048 (<= 256 cells)
//   C. per 256-entry chunk of a cell's list: per-tile counts (warp bit-matrix transpose + popcount)
//   D. per cell: prefix of the chunk counts; one scan over the tiles -> tile_ranges and the pair total
//   E. every chunk writes its splat ids to sorted_ids at (tile start + chunk prefix + rank inside the chunk), ranks
//      from the transposed bit sets in list order, staged so that every run is one coalesced store
// A stable multi-split keeps the depth order inside every tile, so the result equals the oracle's torch.sort(stable)
// of the 64-bit keys element for element (tests/test_gpu_parity.py::test_binning_exact).
//
// Every kernel here is ours, including the device-wide primitives (onesweep.cuh: block and chained scans, onesweep radix passes):
//   phase A  depth_keys (order-preserving compaction of the visible Gaussians through a chained scan; {depth key, id} records
//            + the 32-byte record + the key-byte histograms)  ->  4 onesweep passes over the V visible records
//   phase B  emit_cells (chained scan of the coarse-cell counts in depth order; per-cell histogram)  ->  cell_table (cell
//            ranges, chunk table, digit histograms)  ->  1 onesweep pass by cell (2 above 256 cells)  ->  chunk_counts  ->
//            chunk_prefix  ->  scatter_ids
#include "common.cuh"
#include "onesweep.cuh"

namespace b200gs {

namespace {

constexpr int SUPER_SHIFT = 3;             // coarse cell = 8 x 8 tiles
constexpr int SUPER = 1 << SUPER_SHIFT;
constexpr int CELL_TILES = SUPER * SUPER;  // 64: one bit per tile in a uint64_t mask
constexpr int CHUNK = 256;                 // list entries per block of the count / scatter kernels

// What phase B needs to know about a Gaussian, packed by phase A into ONE 32-byte L2 sector (phase B visits the
// Gaussians in depth order, i.e. at random addresses).
struct __align__(16) SplatRec {
    float x, y, A, B, C, opacity;
    int32_t radius, ncells;
};
static_assert(sizeof(SplatRec) == 32, "SplatRec must be one sector");

// value type of the coarse partition: {tile mask lo, tile mask hi, Gaussian id, unused}
typedef uint4 CellEntry;

constexpr int DEPTH_IPT = 8;                         // records per thread of a depth-sort tile (uint2: 4096 per tile, 32 KB of staging)
constexpr int CELL_IPT = 4;                          // records per thread of a cell-partition tile (uint4: 2048 per tile, 32 KB of staging)
constexpr int DEPTH_TILE = sweep::PASS_THREADS * DEPTH_IPT;
constexpr int CELL_TILE = sweep::PASS_THREADS * CELL_IPT;

constexpr int DK_ITEMS = 8;                          // Gaussians per thread of depth_keys_kernel
constexpr int RO_ITEMS = 8;                          // ranks per thread of rank_offsets_kernel

inline void cell_grid(int width, int height, int& grid_x, int& grid_y, int& cgrid_x, int& cgrid_y) {
    grid_x = div_up(width, TILE);
    grid_y = div_up(height, TILE);
    cgrid_x = div_up(grid_x, SUPER);
    cgrid_y = div_up(grid_y, SUPER);
}

// The sort payload is the Gaussian id; when the id fits 24 bits and a rect can cover at most 255 coarse cells, the cell count of the
// rect rides in the top byte ({key, ncells << 24 | id}): rank_offsets then reads its counts from the sorted records it streams through
// anyway instead of gathering one random 32-byte sector per rank (one L2 request per rank: most of that kernel's time).  Decided from
// (n, width, height) alone, so bin_count and bin_sort agree.
inline bool pack_ncells(int64_t n, int width, int height) {
    int grid_x, grid_y, cgrid_x, cgrid_y;
    cell_grid(width, height, grid_x, grid_y, cgrid_x, cgrid_y);
    return n < (int64_t(1) << 24) && cgrid_x * cgrid_y <= 255;
}
constexpr uint32_t ID_MASK = (1u << 24) - 1u;

// Hands out consecutive 256-byte aligned pieces of a workspace.  With a null base only `off`, the size so far, is meaningful.
struct Carver {
    uintptr_t base;
    size_t off = 0;
    template <typename T>
    T* take(size_t count) {
        T* p = reinterpret_cast<T*>(base + off);
        off = align_up(off + count * sizeof(T), 256);
        return p;
    }
};

// Workspace of phase A (n Gaussians).  Phase B reads the sorted records (rec_a after the four passes) and the 32-byte records.
struct WorkspaceA {
    uint2* rec_a; uint2* rec_b; SplatRec* recs;
    uint32_t* hist; uint32_t* tickets; uint32_t* scan_state; uint32_t* lookback;   // one zero-initialised region of zero_bytes from hist
    size_t zero_bytes, bytes;
    int64_t tiles, blocks;
};

WorkspaceA carve_a(void* base, int64_t n) {
    WorkspaceA W;
    Carver c{reinterpret_cast<uintptr_t>(base)};
    const size_t nn = (size_t)(n > 0 ? n : 1);
    W.tiles = div_up64((int64_t)nn, DEPTH_TILE);
    W.blocks = div_up64((int64_t)nn, 256 * DK_ITEMS);
    W.rec_a = c.take<uint2>(nn);
    W.rec_b = c.take<uint2>(nn);
    W.recs = c.take<SplatRec>(nn);
    const size_t zero = c.off;
    W.hist = c.take<uint32_t>(4 * sweep::RADIX);      // digit histograms, tickets, chained-scan state, look-back words of the 4 passes
    W.tickets = c.take<uint32_t>(16);
    W.scan_state = c.take<uint32_t>((size_t)W.blocks);
    W.lookback = c.take<uint32_t>((size_t)4 * W.tiles * sweep::RADIX);
    W.zero_bytes = c.off - zero;
    W.bytes = c.off;
    return W;
}

// Workspace of phase B (n Gaussians, up to max_coarse coarse entries).
struct WorkspaceB {
    CellEntry* entries_in; CellEntry* entries; uint32_t* offsets;
    uint32_t* cell_hist; uint32_t* tickets; uint32_t* scan_state; uint32_t* lookback;   // one zero-initialised region of zero_bytes from cell_hist
    uint32_t* digit_hist; int2* cell_ranges; int32_t* chunk_base; int32_t* chunk_cell; uint16_t* chunk_cnt; uint32_t* chunk_pre;
    int64_t* tile_start;
    size_t zero_bytes, bytes;
    int64_t max_chunks, tiles, blocks, scan_blocks;
};

WorkspaceB carve_b(void* base, int64_t n, int64_t max_coarse, int width, int height) {
    int grid_x, grid_y, cgrid_x, cgrid_y;
    cell_grid(width, height, grid_x, grid_y, cgrid_x, cgrid_y);
    const size_t n_cells = (size_t)cgrid_x * cgrid_y, n_tiles = (size_t)grid_x * grid_y;
    WorkspaceB W;
    Carver c{reinterpret_cast<uintptr_t>(base)};
    const size_t pp = (size_t)(max_coarse > 0 ? max_coarse : 1), nn = (size_t)(n > 0 ? n : 1);
    W.max_chunks = (int64_t)(pp / CHUNK + n_cells + 1);
    W.tiles = div_up64((int64_t)pp, CELL_TILE);
    W.blocks = div_up64((int64_t)nn, 256);
    W.scan_blocks = div_up64((int64_t)nn, 256 * RO_ITEMS);
    W.entries_in = c.take<CellEntry>(pp);
    W.entries = c.take<CellEntry>(pp);
    W.offsets = c.take<uint32_t>(nn);
    const size_t zero = c.off;
    W.cell_hist = c.take<uint32_t>(n_cells);
    W.tickets = c.take<uint32_t>(16);
    W.scan_state = c.take<uint32_t>((size_t)W.scan_blocks);
    W.lookback = c.take<uint32_t>((size_t)2 * W.tiles * sweep::RADIX);
    W.zero_bytes = c.off - zero;
    W.digit_hist = c.take<uint32_t>(2 * sweep::RADIX);
    W.cell_ranges = c.take<int2>(n_cells);
    W.chunk_base = c.take<int32_t>(n_cells + 1);
    W.chunk_cell = c.take<int32_t>((size_t)W.max_chunks);
    W.chunk_cnt = c.take<uint16_t>((size_t)W.max_chunks * CELL_TILES);
    W.chunk_pre = c.take<uint32_t>((size_t)W.max_chunks * CELL_TILES);
    W.tile_start = c.take<int64_t>(n_tiles);
    W.bytes = c.off;
    return W;
}

// ---- exact tile culling ------------------------------------------------------------------------------------------------
// A (tile, splat) pair can only contribute if some pixel sample p of the tile has alpha = o * exp(-q(p - mu)) >= 1/255,
// q(d) = (A dx^2 + C dy^2)/2 + B dx dy, i.e. if the tile's box of pixel samples meets the ellipse E = {q <= ln(255 o)}.
// E and a tile ROW (a band of 16 sample rows) are convex, so the tiles of that row that meet E are exactly those whose
// sample columns meet the x-extent of (E ∩ band): one interval per row, from two clamped evaluations of the ellipse's
// left/right boundary.  Cost O(rows) per Gaussian instead of O(tiles); every pair dropped would have been skipped by
// the blend loop at all 256 pixels, so images and gradients are bit-identical while the pair list (staging, blend
// evaluations) shrinks ~1.8x on the benchmark scene.  The test only has to be conservative: the threshold carries a
// relative margin of 1e-4 (+1e-3), the interval a 0.01 px slack — orders of magnitude above the error of the
// approximate sqrt used here and of the fp32 / ex2.approx rounding of the blend loop.  Each pair's verdict is computed
// exactly once (emit_cells_kernel) and travels with the pair, so no two kernels ever have to agree on it.
// Per-Gaussian inputs of phase A: separate contiguous arrays xy[n,2], depth[n], radii[n], conic[n,3], opacity[n] (conic and
// opacity NULL without culling), or the columns of one [n,12] row buffer.  Rows may arrive in fixed-size blocks (the sharded
// exchange): block b holds blk_cnt[b] valid rows, the rest of its blk_rows rows is stale memory and reads as culled — no padding
// pass over the receive buffer.
struct BinSrc {
    const float* xy; const float* depth; const int32_t* radii; const float* conic; const float* opacity;
    const int64_t* blk_cnt; int blk_rows;
};

struct CullE {
    float mx, my, B, iA, two_tA, det, ymax, yR;
    int mode;  // 0: full rect (culling off / degenerate conic), 1: spans, 2: nothing visible (opacity <= 1/255)
};

__device__ __forceinline__ CullE make_cull(const SplatRec& r, bool cull) {
    CullE e;
    e.mx = r.x; e.my = r.y;
    e.B = 0.f; e.iA = 1.f; e.two_tA = 0.f; e.det = 1.f; e.ymax = 0.f; e.yR = 0.f;
    e.mode = 0;
    if (!cull) return e;
    const float A = r.A, B = r.B, C = r.C;
    const float o255 = 255.0f * r.opacity;
    if (o255 <= 1.0f) { e.mode = 2; return e; }
    // alpha >= 1/255  <=>  q <= ln(255 o); margin covers every rounding here and in the blend loop
    const float t = __logf(o255) * 1.0001f + 1e-3f;
    const float det = A * C - B * B;
    if (!(det > 0.f) || !(A > 0.f) || !(C > 0.f) || !(t < 3.0e38f)) return e;  // degenerate / NaN: keep the full rect
    const float idet = __frcp_rn(det);
    e.B = B; e.iA = __frcp_rn(A);
    e.two_tA = 2.0f * t * A;
    e.det = det;
    e.ymax = __fsqrt_rn(e.two_tA * idet);
    const float xext = __fsqrt_rn(2.0f * t * C * idet);
    e.yR = -B * xext * __frcp_rn(C);  // the ellipse's rightmost point sits at y = yR, leftmost at -yR
    e.mode = 1;
    return e;
}

__device__ __forceinline__ float sqrt_fast(float x) {
    float r;
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

// tiles [a, b) of tile row ty (clipped to [x0, x1)) whose pixel samples can meet the ellipse
template <bool GSPLAT>
__device__ __forceinline__ bool row_span(const CullE& e, int ty, int x0, int x1, int& a, int& b) {
    a = x0; b = x1;
    if (e.mode == 0) return true;
    const float off = GSPLAT ? 0.5f : 0.0f;
    const float Y0 = float(ty * TILE) + off - e.my;
    const float ya = fmaxf(Y0, -e.ymax), yb = fminf(Y0 + float(TILE - 1), e.ymax);
    if (ya > yb) { b = a; return false; }
    const float yr = fminf(yb, fmaxf(ya, e.yR)), yl = fminf(yb, fmaxf(ya, -e.yR));
    const float dr = sqrt_fast(fmaxf(0.f, e.two_tA - e.det * yr * yr));
    const float dl = sqrt_fast(fmaxf(0.f, e.two_tA - e.det * yl * yl));
    const float xr = (dr - e.B * yr) * e.iA;    // right end of E ∩ band (relative to mu)
    const float xl = (-e.B * yl - dl) * e.iA;   // left end
    // tile tx holds sample columns [16 tx + off, 16 tx + off + 15]
    const float inv = 1.0f / float(TILE);
    const float fa = ceilf((xl + e.mx - (off + float(TILE - 1) + 0.01f)) * inv);
    const float fb = floorf((xr + e.mx - off + 0.01f) * inv);
    if (!(fa <= fb)) {  // also catches NaN
        if (fa == fa && fb == fb) { b = a; return false; }
        return true;    // NaN: keep the whole row
    }
    a = max(x0, (int)fmaxf(fa, -1.0e9f));
    b = min(x1, (int)fminf(fb, 1.0e9f) + 1);
    if (a >= b) { b = a; return false; }
    return true;
}

// tile rect -> rect of coarse cells
__device__ __forceinline__ void coarsen_rect(int x0, int y0, int x1, int y1, int& cx0, int& cy0, int& cx1, int& cy1) {
    cx0 = x0 >> SUPER_SHIFT;
    cy0 = y0 >> SUPER_SHIFT;
    cx1 = ((x1 - 1) >> SUPER_SHIFT) + 1;
    cy1 = ((y1 - 1) >> SUPER_SHIFT) + 1;
}

// Phase A, blocks in ticket order, 2048 consecutive Gaussians per block (the chained scan advances 32..128 blocks per round trip to
// L2, so its length in BLOCKS is what bounds the kernel's latency; 256-Gaussian blocks made it several times slower).  The block
// walks its Gaussians in DK_ITEMS STRIPED rounds (round k, thread t: Gaussian 256 k + t), so every load and the 32-byte record
// stores are coalesced (the first version gave each thread 8 consecutive Gaussians: 384-byte lane stride, 32 sectors per request).
// The visible Gaussians (non-empty tile rect) are compacted in index order into {depth key, id} records: rank = visible Gaussians
// of the rounds before (per-(round, warp) ballot counts, one 64-entry scan) + lanes below in the own ballot + the chained scan over
// the blocks.  Each visible Gaussian gets the 32-byte record phase B works from (indexed by Gaussian id: written right away); the
// histograms of the four key bytes (what the radix passes start from) are accumulated on the way — the two high bytes, which take
// only a handful of values in a scene, with warp-aggregated increments (match.any), the low bytes with plain shared-memory atomics.
// counts[0] += tiles of the rect (the reference's pair count I: an upper bound of the culled count, exact without culling),
// counts[1] += coarse cells, counts[3] = V.
// ROWS: the inputs are the columns of one 16-byte aligned [n,12] row buffer (b200gs.h row layout): three 128-bit loads per Gaussian
template <bool GSPLAT, bool ROWS>
__global__ void __launch_bounds__(256) depth_keys_kernel(int64_t n, int grid_x, int grid_y, int pack, const BinSrc src, uint2* __restrict__ keyrec,
                                                         SplatRec* __restrict__ recs, uint32_t* __restrict__ ticket,
                                                         uint32_t* __restrict__ scan_state, uint32_t* __restrict__ hist,
                                                         unsigned long long* __restrict__ counts) {
    __shared__ unsigned long long s_area[8], s_cells[8];
    __shared__ int s_cnt[DK_ITEMS * 8];      // visible Gaussians of (round, warp); then their exclusive scan
    __shared__ int s_tile;
    __shared__ uint32_t s_excl;
    __shared__ uint32_t s_h[4][sweep::RADIX];
    if (threadIdx.x == 0) s_tile = (int)atomicAdd(ticket, 1u);
    for (int i = threadIdx.x; i < 4 * sweep::RADIX; i += 256) (&s_h[0][0])[i] = 0;
    __syncthreads();
    const int t = s_tile;
    const unsigned lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
    const int64_t base_i = int64_t(t) * (256 * DK_ITEMS) + threadIdx.x;
    unsigned long long area_sum = 0, cell_sum = 0;
    uint32_t key[DK_ITEMS];
    uint32_t hi8[DK_ITEMS];          // pack: the rect's cell count << 24 (rides in the top byte of the sort payload), else 0
    unsigned vis_bits = 0;           // bit k: this thread's Gaussian of round k is visible
    unsigned below[DK_ITEMS];        // visible lanes below this one in round k's ballot
#pragma unroll
    for (int k = 0; k < DK_ITEMS; ++k) {
        const int64_t i = base_i + k * 256;
        key[k] = 0xFFFFFFFFu;
        hi8[k] = 0u;
        bool vis = false;
        if (i < n) {
            float px, py, dep, A = 1.f, B = 0.f, C = 1.f, o = 1.f;
            int r;
            if (ROWS) {
                const float4* row = reinterpret_cast<const float4*>(src.xy + i * B200GS_ROW_FLOATS);
                const float4 q0 = row[0], q1 = row[1], q2 = row[2];
                px = q0.x; py = q0.y; dep = q0.z; A = q0.w; B = q1.x; C = q1.y; o = q1.w;
                r = __float_as_int(q2.w);
                if (src.blk_cnt != nullptr) {
                    const int b = (int)i / src.blk_rows;
                    if ((int)i - b * src.blk_rows >= (int)src.blk_cnt[b]) r = 0;
                }
            } else {
                r = src.radii[i];
                const float2 pp = reinterpret_cast<const float2*>(src.xy)[i];
                px = pp.x; py = pp.y;
                dep = src.depth[i];
                if (src.conic != nullptr) {
                    A = src.conic[3 * i]; B = src.conic[3 * i + 1]; C = src.conic[3 * i + 2];
                    o = src.opacity[i];
                }
            }
            if (r > 0) {
                int x0, y0, x1, y1;
                tile_rect<GSPLAT>(px, py, (float)r, grid_x, grid_y, x0, y0, x1, y1);
                const int area = max(0, x1 - x0) * max(0, y1 - y0);
                if (area > 0) {
                    int cx0, cy0, cx1, cy1;
                    coarsen_rect(x0, y0, x1, y1, cx0, cy0, cx1, cy1);
                    const int ncell = (cx1 - cx0) * (cy1 - cy0);
                    key[k] = __float_as_uint(dep);
                    hi8[k] = pack ? ((uint32_t)ncell << 24) : 0u;
                    area_sum += (unsigned long long)area;
                    cell_sum += (unsigned long long)ncell;
                    vis = true;
                    float4* out = reinterpret_cast<float4*>(recs + i);
                    out[0] = make_float4(px, py, A, B);
                    out[1] = make_float4(C, o, __int_as_float(r), __int_as_float(ncell));
                }
            }
        }
        const unsigned bal = __ballot_sync(0xffffffffu, vis);
        below[k] = __popc(bal & ((1u << lane) - 1u));
        vis_bits |= vis ? (1u << k) : 0u;
        if (lane == 0) s_cnt[k * 8 + w] = __popc(bal);
        // byte histograms: bytes 3 and 2 (few distinct values per scene) warp-aggregated, bytes 1 and 0 with plain atomics
        const unsigned grp = __match_any_sync(0xffffffffu, vis ? (key[k] >> 16) : 0xFFFFFFFFu);
        if (vis) {
            if ((grp & ((1u << lane) - 1u)) == 0u) atomicAdd(&s_h[2][(key[k] >> 16) & 255u], (uint32_t)__popc(grp));
            atomicAdd(&s_h[1][(key[k] >> 8) & 255u], 1u);
            atomicAdd(&s_h[0][key[k] & 255u], 1u);
        }
        const unsigned grp3 = __match_any_sync(0xffffffffu, vis ? (key[k] >> 24) : 0xFFFFFFFFu);
        if (vis && (grp3 & ((1u << lane) - 1u)) == 0u) atomicAdd(&s_h[3][key[k] >> 24], (uint32_t)__popc(grp3));
    }
    __syncthreads();
    if (threadIdx.x < 32) {     // warp 0: scan of the 64 (round, warp) counts, then the warp-wide look-back over the preceding blocks
        const int c0 = s_cnt[2 * lane], c1 = s_cnt[2 * lane + 1];
        const int inc = sweep::warp_inclusive(c0 + c1);
        const int block_vis = __shfl_sync(0xffffffffu, inc, 31);
        s_cnt[2 * lane] = inc - c0 - c1;
        s_cnt[2 * lane + 1] = inc - c1;
        const uint32_t excl = sweep::chained_exclusive(scan_state, t, (uint32_t)block_vis);
        if (threadIdx.x == 0) {
            s_excl = excl;
            if (t == (int)gridDim.x - 1) counts[3] = (unsigned long long)(excl + (uint32_t)block_vis);
        }
    }
    __syncthreads();
    const uint32_t base = s_excl;
#pragma unroll
    for (int k = 0; k < DK_ITEMS; ++k) {
        if (!((vis_bits >> k) & 1u)) continue;
        keyrec[base + (uint32_t)s_cnt[k * 8 + w] + below[k]] = make_uint2(key[k], (uint32_t)(base_i + k * 256) | hi8[k]);
    }
    unsigned long long a = area_sum, c = cell_sum;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, o);
        c += __shfl_xor_sync(0xffffffffu, c, o);
    }
    if ((threadIdx.x & 31) == 0) { s_area[threadIdx.x >> 5] = a; s_cells[threadIdx.x >> 5] = c; }
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long ta = 0, tc = 0;
#pragma unroll
        for (int w2 = 0; w2 < 8; ++w2) { ta += s_area[w2]; tc += s_cells[w2]; }
        if (ta) atomicAdd(counts, ta);
        if (tc) atomicAdd(counts + 1, tc);
    }
    for (int i = threadIdx.x; i < 4 * sweep::RADIX; i += 256) {
        const uint32_t v = (&s_h[0][0])[i];
        if (v) atomicAdd(hist + i, v);
    }
}

// Exclusive prefix of the coarse-cell counts over the depth-ranked Gaussians: offsets[rank] = first entry slot of that rank.  Big
// tiles (RO_ITEMS consecutive ranks per thread) for the same reason as above; the cell count of a rank is gathered from its record.
__global__ void __launch_bounds__(256) rank_offsets_kernel(const int64_t* __restrict__ d_visible, int pack, const uint2* __restrict__ order,
                                                          const SplatRec* __restrict__ recs, uint32_t* __restrict__ offsets,
                                                          uint32_t* __restrict__ ticket, uint32_t* __restrict__ scan_state) {
    const int t = sweep::block_ticket(ticket);
    const int64_t n = *d_visible;
    const int64_t r0 = (int64_t(t) * blockDim.x + threadIdx.x) * RO_ITEMS;
    if (int64_t(t) * blockDim.x * RO_ITEMS >= n) return;
    int nc[RO_ITEMS];
    int mine = 0;
#pragma unroll
    for (int k = 0; k < RO_ITEMS; ++k) {
        nc[k] = 0;
        if (r0 + k < n) {
            const uint32_t y = order[r0 + k].y;
            nc[k] = pack ? (int)(y >> 24) : __ldg(&recs[y].ncells);
        }
        mine += nc[k];
    }
    uint32_t run = sweep::chained_block_exclusive<8>(mine, scan_state, t);
#pragma unroll
    for (int k = 0; k < RO_ITEMS; ++k) {
        if (r0 + k < n) offsets[r0 + k] = run;
        run += (uint32_t)nc[k];
    }
}

// Phase B, one block (in ticket order) per 256 depth-ranked Gaussians: emits their (coarse cell, {tile mask, id}) entries, cells
// in row-major order.  The first slot of a rank is the exclusive prefix of the cell counts in depth order: block scan +
// chained scan over the blocks, so the block's ranks own one contiguous window of the entry array; the entries are
// assembled in shared memory and written back with coalesced stores.  The expensive part — one ellipse/row-band
// intersection per tile row of every rect — is spread over the block as (rank, row) work items, so a warp never waits
// for the one lane that owns a large splat.  The block also counts its entries per cell (the histogram the partition and
// the cell ranges are derived from).
constexpr int EMIT_SLOTS = 2048;
constexpr int EMIT_ITEMS = 2048;  // (rank, row) work items resolved through a table instead of a binary search
constexpr int EMIT_HIST = 1024;   // cells counted in shared memory (images up to 4096 x 4096); larger grids count straight in global memory

template <bool GSPLAT>
__global__ void __launch_bounds__(256) emit_cells_kernel(const int64_t* __restrict__ d_visible, int pack, int grid_x, int grid_y, int cgrid_x, int cull,
                                                         int64_t max_coarse, const uint2* __restrict__ order, const SplatRec* __restrict__ recs,
                                                         const uint32_t* __restrict__ offsets, CellEntry* __restrict__ entries, int n_cells,
                                                         uint32_t* __restrict__ cell_hist) {
    __shared__ unsigned short s_k[EMIT_SLOTS];
    __shared__ int32_t s_id[EMIT_SLOTS];
    __shared__ unsigned long long s_mask[EMIT_SLOTS];
    __shared__ float s_f[8][256];        // mx, my, B, iA, two_tA, det, ymax, yR
    __shared__ int s_mode[256], s_xr[256], s_yr[256], s_start[256];   // x0 | x1 << 16, y0 | y1 << 16, first slot - block_lo
    __shared__ int s_rowoff[256];
    __shared__ unsigned char s_item[EMIT_ITEMS];   // work item -> rank of the block (when the block has <= EMIT_ITEMS tile rows)
    __shared__ int s_warp[9];
    __shared__ uint32_t s_hist[EMIT_HIST];
    const int tid = threadIdx.x;
    const int64_t n = *d_visible;
    const int64_t rank0 = int64_t(blockIdx.x) * blockDim.x;
    if (rank0 >= n) return;
    const bool smem_hist = n_cells <= EMIT_HIST;
    if (smem_hist)
        for (int i = tid; i < n_cells; i += 256) s_hist[i] = 0;
    const int64_t rnk = rank0 + tid;
    int g = -1, x0 = 0, y0 = 0, x1 = 0, y1 = 0, t = 0, nrows = 0;
    CullE e{};
    if (rnk < n) {
        g = (int)(pack ? (order[rnk].y & ID_MASK) : order[rnk].y);
        const float4* rp = reinterpret_cast<const float4*>(recs + g);
        const float4 r0 = __ldg(rp), r1 = __ldg(rp + 1);
        SplatRec rec;
        rec.x = r0.x; rec.y = r0.y; rec.A = r0.z; rec.B = r0.w; rec.C = r1.x; rec.opacity = r1.y;
        rec.radius = __float_as_int(r1.z); rec.ncells = __float_as_int(r1.w);
        t = rec.ncells;
        if (t > 0) {
            tile_rect<GSPLAT>(rec.x, rec.y, (float)rec.radius, grid_x, grid_y, x0, y0, x1, y1);
            e = make_cull(rec, cull != 0);
            nrows = (e.mode == 2) ? 0 : y1 - y0;
        }
    }
    // first slot of this rank = cells of the ranks before it (rank_offsets_kernel); the block's ranks own one contiguous window
    const int64_t block_lo = (int64_t)offsets[rank0];
    const int64_t last_rank = min(rank0 + (int64_t)blockDim.x, n) - 1;
    const uint32_t last_y = order[last_rank].y;
    const int block_cells = (int)((int64_t)offsets[last_rank] + (pack ? (int)(last_y >> 24) : __ldg(&recs[last_y].ncells)) - block_lo);
    const int local_start = (rnk < n) ? (int)((int64_t)offsets[rnk] - block_lo) : block_cells;
    int total_rows;
    s_rowoff[tid] = sweep::block_exclusive<int, 8>(nrows, s_warp, &total_rows);   // exclusive scan of the row counts
    s_f[0][tid] = e.mx; s_f[1][tid] = e.my; s_f[2][tid] = e.B; s_f[3][tid] = e.iA;
    s_f[4][tid] = e.two_tA; s_f[5][tid] = e.det; s_f[6][tid] = e.ymax; s_f[7][tid] = e.yR;
    s_mode[tid] = e.mode;
    s_xr[tid] = x0 | (x1 << 16);
    s_yr[tid] = y0 | (y1 << 16);
    s_start[tid] = local_start;
    const int cx0 = x0 >> SUPER_SHIFT, cy0 = y0 >> SUPER_SHIFT;
    const int cw = t > 0 ? ((x1 - 1) >> SUPER_SHIFT) - cx0 + 1 : 1;
    __syncthreads();
    const bool item_table = total_rows <= EMIT_ITEMS;
    if (item_table) {     // rank tid owns items [s_rowoff[tid], s_rowoff[tid] + nrows)
        const int o = s_rowoff[tid];
        for (int k = 0; k < nrows; ++k) s_item[o + k] = (unsigned char)tid;
    }                     // visible to the item loop after the barrier that follows the cell/id stores below
    const int64_t block_hi = min(block_lo + block_cells, max_coarse);
    for (int64_t lo = block_lo; lo < block_hi; lo += EMIT_SLOTS) {
        const int cn = (int)min((int64_t)EMIT_SLOTS, block_hi - lo);
        const int wlo = (int)(lo - block_lo);       // window = local slots [wlo, wlo + cn)
        for (int i = tid; i < cn; i += 256) s_mask[i] = 0ull;
        // cells and ids of this rank's slots
        {
            const int ls = local_start;
            int k = max(0, wlo - ls);
            const int kend = min(t, wlo + cn - ls);
            int cy = cy0 + k / cw, cx = cx0 + k % cw;
            for (; k < kend; ++k) {
                const int cell = cy * cgrid_x + cx;
                s_k[ls + k - wlo] = (unsigned short)cell;
                s_id[ls + k - wlo] = g;
                if (smem_hist) atomicAdd(&s_hist[cell], 1u); else atomicAdd(cell_hist + cell, 1u);
                if (++cx == cx0 + cw) { cx = cx0; ++cy; }
            }
        }
        __syncthreads();
        // (rank, row) work items
        for (int it = tid; it < total_rows; it += 256) {
            int r = 0;
            if (item_table) {
                r = s_item[it];
            } else {
#pragma unroll
                for (int step = 128; step >= 1; step >>= 1)
                    if (s_rowoff[r + step] <= it) r += step;
            }
            CullE q;
            q.mx = s_f[0][r]; q.my = s_f[1][r]; q.B = s_f[2][r]; q.iA = s_f[3][r];
            q.two_tA = s_f[4][r]; q.det = s_f[5][r]; q.ymax = s_f[6][r]; q.yR = s_f[7][r];
            q.mode = s_mode[r];
            const int xr = s_xr[r], yr = s_yr[r];
            const int rx0 = xr & 0xffff, rx1 = xr >> 16, ry0 = yr & 0xffff;
            const int ty = ry0 + (it - s_rowoff[r]);
            int a, b;
            if (!row_span<GSPLAT>(q, ty, rx0, rx1, a, b)) continue;
            const int rcx0 = rx0 >> SUPER_SHIFT, rcw = ((rx1 - 1) >> SUPER_SHIFT) - rcx0 + 1;
            const int row_slot = s_start[r] + ((ty >> SUPER_SHIFT) - (ry0 >> SUPER_SHIFT)) * rcw - rcx0 - wlo;
            for (int cx = a >> SUPER_SHIFT; cx <= (b - 1) >> SUPER_SHIFT; ++cx) {
                const int slot = row_slot + cx;
                if (slot < 0 || slot >= cn) continue;
                const int wx0 = cx << SUPER_SHIFT;
                const int ca = max(a, wx0) - wx0, cb = min(b, wx0 + SUPER) - wx0;
                const unsigned bits = ((1u << (cb - ca)) - 1u) << ca;
                reinterpret_cast<unsigned char*>(s_mask)[slot * 8 + (ty & (SUPER - 1))] = (unsigned char)bits;
            }
        }
        __syncthreads();
        for (int i = tid; i < cn; i += 256) {
            const unsigned long long m = s_mask[i];
            entries[lo + i] = make_uint4((uint32_t)m, (uint32_t)(m >> 32), (uint32_t)s_id[i], (uint32_t)s_k[i]);
        }
        __syncthreads();
    }
    if (smem_hist)
        for (int i = tid; i < n_cells; i += 256) {
            const uint32_t c = s_hist[i];
            if (c) atomicAdd(cell_hist + i, c);
        }
}

// One block, after the emit: from the per-cell entry counts -> cell ranges (exclusive scan), the chunk table
// (chunk_base[c] = number of CHUNK-entry chunks of the cells before c; chunk_cell[chunk] = its cell), the digit histograms
// of the partition passes (low / high byte of the cell id), zeroed tile totals.
__global__ void __launch_bounds__(1024) cell_table_kernel(int n_cells, const uint32_t* __restrict__ cell_hist, int2* __restrict__ cell_ranges,
                                                          int32_t* __restrict__ chunk_base, int32_t* __restrict__ chunk_cell,
                                                          uint32_t* __restrict__ digit_hist, int n_tiles, int64_t* __restrict__ tile_total) {
    __shared__ int s_warp[33];
    __shared__ uint32_t s_dh[2][sweep::RADIX];
    const int tid = threadIdx.x;
    for (int i = tid; i < 2 * sweep::RADIX; i += 1024) (&s_dh[0][0])[i] = 0;
    __syncthreads();
    int total = 0, entries = 0;     // chunks / entries of the cells before this round
    for (int base = 0; base < n_cells; base += 1024) {
        const int i = base + tid;
        int cnt = 0, v = 0;
        if (i < n_cells) {
            cnt = (int)cell_hist[i];
            v = (cnt + CHUNK - 1) / CHUNK;
            if (cnt) { atomicAdd(&s_dh[0][i & 255], (uint32_t)cnt); atomicAdd(&s_dh[1][(i >> 8) & 255], (uint32_t)cnt); }
        }
        int round_chunks, round_entries;
        const int excl = total + sweep::block_exclusive<int, 32>(v, s_warp, &round_chunks);
        const int excl2 = entries + sweep::block_exclusive<int, 32>(cnt, s_warp, &round_entries);
        if (i < n_cells) {
            chunk_base[i] = excl;
            cell_ranges[i] = cnt > 0 ? make_int2(excl2, excl2 + cnt) : make_int2(0, 0);
        }
        total += round_chunks;
        entries += round_entries;
    }
    if (tid == 0) chunk_base[n_cells] = total;
    for (int i = tid; i < 2 * sweep::RADIX; i += 1024) digit_hist[i] = (&s_dh[0][0])[i];
    for (int i = tid; i < n_tiles; i += 1024) tile_total[i] = 0;    // accumulated by chunk_counts_kernel
    __syncthreads();                                                // chunk_base (written by this block) is visible
    __shared__ int s_cb[1024];                                      // chunk_base of up to 1024 cells (images up to 4096 x 4096): the
    const bool in_smem = n_cells <= 1024;                           // binary search below is a chain of dependent loads per chunk
    if (in_smem) {
        if (tid < n_cells) s_cb[tid] = chunk_base[tid];
        __syncthreads();
    }
    for (int c = tid; c < total; c += 1024) {
        int lo = 0, hi = n_cells;   // invariant: chunk_base[lo] <= c < chunk_base[hi]; cells without entries own no chunk
        while (hi - lo > 1) {
            const int mid = (lo + hi) >> 1;
            if ((in_smem ? s_cb[mid] : chunk_base[mid]) <= c) lo = mid; else hi = mid;
        }
        chunk_cell[c] = lo;
    }
}

// 32x32 bit-matrix transpose across a warp: lane l passes row l, lane t receives column t
// (bit l of the result = bit t of lane l's input).
__device__ __forceinline__ uint32_t transpose32(uint32_t x, unsigned lane) {
#pragma unroll
    for (int j = 16; j >= 1; j >>= 1) {
        const uint32_t m = (j == 16) ? 0x0000FFFFu : (j == 8) ? 0x00FF00FFu : (j == 4) ? 0x0F0F0F0Fu : (j == 2) ? 0x33333333u : 0x55555555u;
        const uint32_t y = __shfl_xor_sync(0xffffffffu, x, j);
        x = (lane & j) ? ((x & ~m) | ((y >> j) & m)) : ((x & m) | ((y << j) & ~m));
    }
    return x;
}

// Prologue of phases C and E, one block per chunk c (CHUNK consecutive entries of one cell's depth-ordered list): thread i loads
// entry i of the chunk (with IDS it also stores its Gaussian id to s_id[i]; without, it reads the masks only: half the bytes).
// Each warp transposes the masks of its 32 entries: lane t then holds in wlo / whi, for tiles t and t+32, the bit set of the
// warp's entries that reach the tile, and s_cnt[warp][tile] = its popcount.  Returns the chunk's cell.
template <bool IDS>
__device__ __forceinline__ int load_chunk(int c, const int2* __restrict__ cell_ranges, const int32_t* __restrict__ chunk_base,
                                          const int32_t* __restrict__ chunk_cell, const CellEntry* __restrict__ entries,
                                          uint16_t (*s_cnt)[CELL_TILES], int32_t* s_id, uint32_t& wlo, uint32_t& whi) {
    const int cell = __ldg(chunk_cell + c);
    const int2 r = cell_ranges[cell];
    const int e = r.x + (c - __ldg(chunk_base + cell)) * CHUNK + (int)threadIdx.x;
    const unsigned lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
    uint32_t lo = 0, hi = 0;
    if (e < r.y) {
        if (IDS) {
            const uint4 v = __ldg(entries + e);
            lo = v.x; hi = v.y;
            s_id[threadIdx.x] = (int)v.z;
        } else {
            const uint2 m = __ldg(reinterpret_cast<const uint2*>(entries + e));
            lo = m.x; hi = m.y;
        }
    }
    wlo = transpose32(lo, lane);
    whi = transpose32(hi, lane);
    s_cnt[w][lane] = (uint16_t)__popc(wlo);
    s_cnt[w][lane + 32] = (uint16_t)__popc(whi);
    return cell;
}

// tile t of a coarse cell (bit t of its masks) -> tile coordinates
__device__ __forceinline__ int2 cell_tile(int cell, int t, int cgrid_x) {
    return make_int2(((cell % cgrid_x) << SUPER_SHIFT) + (t & (SUPER - 1)), ((cell / cgrid_x) << SUPER_SHIFT) + (t >> SUPER_SHIFT));
}

// Phase C: per-tile entry counts of every chunk.
__global__ void __launch_bounds__(CHUNK) chunk_counts_kernel(int n_cells, int cgrid_x, int grid_x, int grid_y, const int2* __restrict__ cell_ranges,
                                                             const int32_t* __restrict__ chunk_base, const int32_t* __restrict__ chunk_cell,
                                                             const CellEntry* __restrict__ entries, uint16_t* __restrict__ chunk_cnt,
                                                             int64_t* __restrict__ tile_total) {
    __shared__ uint16_t s_cnt[CHUNK / 32][CELL_TILES];
    const int c = blockIdx.x;
    if (c >= __ldg(chunk_base + n_cells)) return;
    uint32_t wlo, whi;
    const int cell = load_chunk<false>(c, cell_ranges, chunk_base, chunk_cell, entries, s_cnt, nullptr, wlo, whi);
    __syncthreads();
    if (threadIdx.x < CELL_TILES) {
        int sum = 0;
#pragma unroll
        for (int k = 0; k < CHUNK / 32; ++k) sum += s_cnt[k][threadIdx.x];
        chunk_cnt[int64_t(c) * CELL_TILES + threadIdx.x] = (uint16_t)sum;
        const int2 tile = cell_tile(cell, threadIdx.x, cgrid_x);
        if (sum > 0 && tile.x < grid_x && tile.y < grid_y)
            atomicAdd(reinterpret_cast<unsigned long long*>(tile_total + int64_t(tile.y) * grid_x + tile.x), (unsigned long long)sum);
    }
}

// Phase D.  Blocks [0, n_cells): thread (j, t) of a cell's block computes the prefix over the cell's chunks of tile t's
// counts, the chunk list split into 16 contiguous parts j so that the sequential walks stay short.  Block n_cells, at the
// same time: exclusive scan of the tile totals (accumulated by chunk_counts_kernel) in tile-id order, in place -> tile
// starts; tile_ranges (clamped to the capacity of sorted_ids; empty tiles (0,0) like dgr's zero-filled ranges); counts[2].
__global__ void __launch_bounds__(1024) chunk_prefix_kernel(int n_cells, int n_tiles, const int32_t* __restrict__ chunk_base,
                                                            const uint16_t* __restrict__ chunk_cnt, uint32_t* __restrict__ chunk_pre,
                                                            int64_t* __restrict__ tile_start, int64_t max_pairs,
                                                            int2* __restrict__ tile_ranges, int64_t* __restrict__ d_counts) {
    __shared__ uint32_t s_part[16][CELL_TILES];
    __shared__ int64_t s_warp[32];
    __shared__ int64_t s_carry;     // pairs of the tiles before this round
    const int tid = threadIdx.x;
    if ((int)blockIdx.x < n_cells) {
        const int cell = blockIdx.x;
        const int t = tid & (CELL_TILES - 1), j = tid >> 6;
        const int c0 = chunk_base[cell], c1 = chunk_base[cell + 1];
        const int per = (c1 - c0 + 15) >> 4;
        const int a = min(c1, c0 + j * per), b = min(c1, a + per);
        // the walk is a chain of dependent L2 round trips unless the loads are issued together: up to PRE_REG counts per thread live in
        // registers (all loads in flight at once, read once), longer parts fall back to the two-pass loop
        constexpr int PRE_REG = 16;
        uint32_t sum = 0;
        if (per <= PRE_REG) {
            uint32_t v[PRE_REG];
#pragma unroll
            for (int q = 0; q < PRE_REG; ++q) v[q] = (a + q < b) ? (uint32_t)chunk_cnt[int64_t(a + q) * CELL_TILES + t] : 0u;
#pragma unroll
            for (int q = 0; q < PRE_REG; ++q) sum += v[q];
            s_part[j][t] = sum;
            __syncthreads();
            uint32_t run = 0;
            for (int k = 0; k < j; ++k) run += s_part[k][t];
#pragma unroll
            for (int q = 0; q < PRE_REG; ++q) {
                if (a + q < b) chunk_pre[int64_t(a + q) * CELL_TILES + t] = run;
                run += v[q];
            }
            return;
        }
#pragma unroll 4
        for (int c = a; c < b; ++c) sum += chunk_cnt[int64_t(c) * CELL_TILES + t];
        s_part[j][t] = sum;
        __syncthreads();
        uint32_t run = 0;
        for (int k = 0; k < j; ++k) run += s_part[k][t];
#pragma unroll 4
        for (int c = a; c < b; ++c) {
            const uint32_t v = chunk_cnt[int64_t(c) * CELL_TILES + t];
            chunk_pre[int64_t(c) * CELL_TILES + t] = run;
            run += v;
        }
        return;
    }
    if (tid == 0) s_carry = 0;
    for (int base = 0; base < n_tiles; base += 8192) {
        const int i0 = base + tid * 8;
        int64_t v[8];
        if (i0 + 8 <= n_tiles) {
            const longlong2* p = reinterpret_cast<const longlong2*>(tile_start + i0);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const longlong2 q = p[k];
                v[2 * k] = q.x; v[2 * k + 1] = q.y;
            }
        } else {
#pragma unroll
            for (int k = 0; k < 8; ++k) v[k] = (i0 + k < n_tiles) ? tile_start[i0 + k] : 0;
        }
        int64_t sum = 0;
#pragma unroll
        for (int k = 0; k < 8; ++k) sum += v[k];
        int64_t run = sweep::block_exclusive<int64_t, 32>(sum, s_warp, nullptr);
        run += s_carry;     // after the scan's barriers: the carry of the rounds before
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            if (i0 + k < n_tiles) {
                tile_start[i0 + k] = run;
                tile_ranges[i0 + k] = v[k] > 0 ? make_int2((int)min(run, max_pairs), (int)min(run + v[k], max_pairs)) : make_int2(0, 0);
            }
            run += v[k];
        }
        __syncthreads();    // every thread has read s_carry
        if (tid == 1023) s_carry = run;
        __syncthreads();
    }
    if (tid == 0) d_counts[2] = s_carry;
}

// Phase E: one block per chunk; sorted_ids[tile start + chunk prefix + rank in chunk] = id.  After the warp transpose,
// lane t owns the bit sets of tiles t / t+32 over the warp's 32 entries; walking their set bits in order yields the
// tile's ids in list order.  The chunk's output is first laid out in shared memory in (tile, rank) order — the order it
// has in global memory, where tile t's part is one contiguous run — so each run leaves the SM as one coalesced store
// instead of one partial-sector write per id.
constexpr int SCATTER_STAGE = 4096;

__global__ void __launch_bounds__(CHUNK) scatter_ids_kernel(int n_cells, int cgrid_x, int grid_x, int grid_y, int64_t max_pairs,
                                                            const int2* __restrict__ cell_ranges, const int32_t* __restrict__ chunk_base,
                                                            const int32_t* __restrict__ chunk_cell, const CellEntry* __restrict__ entries,
                                                            const uint32_t* __restrict__ chunk_pre, const int64_t* __restrict__ tile_start,
                                                            int32_t* __restrict__ sorted_ids) {
    constexpr int WARPS = CHUNK / 32;
    __shared__ uint16_t s_cnt[WARPS][CELL_TILES];
    __shared__ int s_wbase[WARPS][CELL_TILES];    // offset of (warp, tile) inside the tile's run of this chunk
    __shared__ int s_off[CELL_TILES + 1];         // offset of tile t's run inside the staged output
    __shared__ int64_t s_gbase[CELL_TILES];       // global position of tile t's run
    __shared__ int32_t s_id[CHUNK];
    __shared__ int32_t s_out[SCATTER_STAGE];
    const int c = blockIdx.x;
    if (c >= __ldg(chunk_base + n_cells)) return;
    const unsigned lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
    uint32_t wlo, whi;     // entries of this warp reaching tile lane / lane + 32
    const int cell = load_chunk<true>(c, cell_ranges, chunk_base, chunk_cell, entries, s_cnt, s_id, wlo, whi);
    __syncthreads();
    if (threadIdx.x < CELL_TILES) {
        const int t = threadIdx.x;
        const int2 tile = cell_tile(cell, t, cgrid_x);
        s_gbase[t] = (tile.x < grid_x && tile.y < grid_y) ? tile_start[int64_t(tile.y) * grid_x + tile.x] + chunk_pre[int64_t(c) * CELL_TILES + t] : 0;
        int run = 0;
#pragma unroll
        for (int k = 0; k < WARPS; ++k) {
            s_wbase[k][t] = run;
            run += s_cnt[k][t];
        }
        s_off[t + 1] = sweep::warp_inclusive(run);   // inclusive scan of the tile totals inside each of the two warps
    }
    __syncthreads();
    const int half = s_off[32];       // total of tiles 0..31
    __syncthreads();
    if (threadIdx.x >= 32 && threadIdx.x < CELL_TILES) s_off[threadIdx.x + 1] += half;
    if (threadIdx.x == 0) s_off[0] = 0;
    __syncthreads();
    const int total = s_off[CELL_TILES];
    const int32_t* ids = s_id + w * 32;
    if (total <= SCATTER_STAGE) {
        int p = s_off[lane] + s_wbase[w][lane];
        for (; wlo; wlo &= wlo - 1) s_out[p++] = ids[__ffs(wlo) - 1];
        p = s_off[lane + 32] + s_wbase[w][lane + 32];
        for (; whi; whi &= whi - 1) s_out[p++] = ids[__ffs(whi) - 1];
        __syncthreads();
        for (int t = (int)w; t < CELL_TILES; t += WARPS) {     // warp w flushes the runs of tiles w, w+8, ...
            const int o = s_off[t], len = s_off[t + 1] - o;
            const int64_t gb = s_gbase[t];
            for (int k = (int)lane; k < len; k += 32)
                if (gb + k < max_pairs) sorted_ids[gb + k] = s_out[o + k];
        }
    } else {   // a chunk of very large splats: write straight to global memory
        int64_t p = s_gbase[lane] + s_wbase[w][lane];
        for (; wlo; wlo &= wlo - 1, ++p)
            if (p < max_pairs) sorted_ids[p] = ids[__ffs(wlo) - 1];
        p = s_gbase[lane + 32] + s_wbase[w][lane + 32];
        for (; whi; whi &= whi - 1, ++p)
            if (p < max_pairs) sorted_ids[p] = ids[__ffs(whi) - 1];
    }
}

}  // namespace

// Counter read-back.  For pinned (mapped) host memory the counters are PUBLISHED by a kernel with system-scope stores
// instead of a cudaMemcpyAsync: an in-stream D2H copy is serviced by a copy engine, and queues behind whatever bulk
// transfer the application has in flight on it (e.g. the H2D prefetch of the next training image) — which would stall
// the whole forward behind a 32-byte copy.  Pageable host memory falls back to the copy.
__global__ void publish_i64_kernel(const int64_t* __restrict__ src, volatile int64_t* __restrict__ dst, int n) {
    for (int i = threadIdx.x; i < n; i += blockDim.x) dst[i] = src[i];
    __threadfence_system();
}

static int publish_i64(const int64_t* d_values, int64_t* host_values, int n, cudaStream_t s) {
    cudaPointerAttributes attr{};
    const cudaError_t e = cudaPointerGetAttributes(&attr, host_values);
    if (e == cudaSuccess && attr.type == cudaMemoryTypeHost && attr.devicePointer != nullptr) {
        publish_i64_kernel<<<1, 32, 0, s>>>(d_values, (volatile int64_t*)attr.devicePointer, n);   // one warp: every warp pays for a fence
        B200GS_LAUNCH_CHECK();
    } else {
        (void)cudaGetLastError();
        B200GS_CUDA(cudaMemcpyAsync(host_values, d_values, sizeof(int64_t) * (size_t)n, cudaMemcpyDeviceToHost, s));
    }
    return B200GS_OK;
}

// the four binning counters to host_counts (when given), then optionally wait for them
static int publish_counts(const int64_t* d_counts, int64_t* host_counts, int sync_host, cudaStream_t s) {
    if (host_counts == nullptr) return B200GS_OK;
    const int rc = publish_i64(d_counts, host_counts, 4, s);
    if (rc != B200GS_OK) return rc;
    if (sync_host) B200GS_CUDA(cudaStreamSynchronize(s));
    return B200GS_OK;
}

// The count stage of both entry points.  rows: xy, depth, radii, conic and opacity are columns of one 16-byte aligned [n,12] row
// buffer (b200gs.h), optionally in blocks of block_rows rows of which the first block_counts[b] are valid; otherwise separate
// arrays, conic and opacity NULL without culling
static int bin_count(int mode, int width, int height, int64_t n, bool rows, const float* xy, const float* depth, const int32_t* radii,
                     const float* conic, const float* opacity, void* ws, size_t ws_bytes, int64_t* d_counts, int64_t* host_counts,
                     int sync_host, cudaStream_t s, const int64_t* block_counts = nullptr, int64_t block_rows = 0) {
    const WorkspaceA W = carve_a(ws, n);
    if (ws_bytes < W.bytes) {
        set_error("bin_count: workspace too small (%zu < %zu)", ws_bytes, W.bytes);
        return B200GS_ENOSPACE;
    }
    if (n >= (int64_t(1) << 30)) {
        set_error("bin_count: %lld Gaussians exceed the 2^30 limit of the look-back words", (long long)n);
        return B200GS_ENOSPACE;
    }
    const int grid_x = div_up(width, TILE), grid_y = div_up(height, TILE);
    B200GS_CUDA(cudaMemsetAsync(d_counts, 0, 4 * sizeof(int64_t), s));
    if (n > 0) {
        B200GS_CUDA(cudaMemsetAsync(W.hist, 0, W.zero_bytes, s));
        const BinSrc src{xy, depth, radii, conic, opacity, block_rows > 0 ? block_counts : nullptr, (int)block_rows};
        const int pack = pack_ncells(n, width, height) ? 1 : 0;
        static constexpr decltype(&depth_keys_kernel<false, false>) kernels[2][2] = {
            {depth_keys_kernel<false, false>, depth_keys_kernel<false, true>}, {depth_keys_kernel<true, false>, depth_keys_kernel<true, true>}};
        kernels[mode == B200GS_MODE_GSPLAT][rows]<<<(unsigned)W.blocks, 256, 0, s>>>(n, grid_x, grid_y, pack, src, W.rec_a, W.recs, W.tickets,
                                                                                   W.scan_state, W.hist, (unsigned long long*)d_counts);
        B200GS_LAUNCH_CHECK();
        // stable LSD sort of the V visible {depth key, id} records (V = d_counts[3], known on the device only; byte histograms from above)
        const int64_t* d_visible = d_counts + 3;
        uint2* src_rec = W.rec_a;
        uint2* dst_rec = W.rec_b;
        for (int pass = 0; pass < 4; ++pass) {
            sweep::onesweep_pass_kernel<uint2, DEPTH_IPT><<<(unsigned)W.tiles, sweep::PASS_THREADS, 0, s>>>(
                src_rec, dst_rec, d_visible, n, 8 * pass, W.hist + pass * sweep::RADIX, W.lookback + (size_t)pass * W.tiles * sweep::RADIX,
                W.tickets + 1 + pass);
            B200GS_LAUNCH_CHECK();
            uint2* tmp = src_rec; src_rec = dst_rec; dst_rec = tmp;
        }
        // 4 passes: the sorted records are back in rec_a
    }
    return publish_counts(d_counts, host_counts, sync_host, s);
}

// ---- row packing for the Gaussian-sharded exchange -------------------------------------------------------------------
namespace {

// scan[i] = number of entries with radius > 0 before i: block scan + chained scan over the blocks (ticket order).  VS_ITEMS
// consecutive entries per thread: the chained scan's latency is its length in BLOCKS (with 256-entry blocks the 11.7 k blocks
// of a 3 M-entry scan made this kernel most of the pack stage).
constexpr int VS_ITEMS = 8;

__global__ void __launch_bounds__(256) visible_scan_kernel(int64_t n, const int32_t* __restrict__ radii, int32_t* __restrict__ scan,
                                                           uint32_t* __restrict__ ticket, uint32_t* __restrict__ state) {
    const int t = sweep::block_ticket(ticket);
    const int64_t i0 = (int64_t(t) * blockDim.x + threadIdx.x) * VS_ITEMS;
    int vis[VS_ITEMS];
    int mine = 0;
    const bool vec = i0 + VS_ITEMS <= n && (reinterpret_cast<uintptr_t>(radii) & 15u) == 0;    // i0 is a multiple of 8
    if (vec) {
        const int4 a = __ldg(reinterpret_cast<const int4*>(radii + i0)), b = __ldg(reinterpret_cast<const int4*>(radii + i0) + 1);
        vis[0] = a.x > 0; vis[1] = a.y > 0; vis[2] = a.z > 0; vis[3] = a.w > 0;
        vis[4] = b.x > 0; vis[5] = b.y > 0; vis[6] = b.z > 0; vis[7] = b.w > 0;
    } else {
#pragma unroll
        for (int k = 0; k < VS_ITEMS; ++k) vis[k] = (i0 + k < n && radii[i0 + k] > 0) ? 1 : 0;
    }
#pragma unroll
    for (int k = 0; k < VS_ITEMS; ++k) mine += vis[k];
    int run = (int)sweep::chained_block_exclusive<8>(mine, state, t);
    int out[VS_ITEMS];
#pragma unroll
    for (int k = 0; k < VS_ITEMS; ++k) { out[k] = run; run += vis[k]; }
    if (vec) {                       // scan is the library's own workspace: aligned
        reinterpret_cast<int4*>(scan + i0)[0] = make_int4(out[0], out[1], out[2], out[3]);
        reinterpret_cast<int4*>(scan + i0)[1] = make_int4(out[4], out[5], out[6], out[7]);
    } else {
#pragma unroll
        for (int k = 0; k < VS_ITEMS; ++k)
            if (i0 + k < n) scan[i0 + k] = out[k];
    }
}

// scan[i] = number of visible entries before i = the row of entry i (row_index[i], what the backward uses to find entry i's
// gradient row); *d_count = total.
__global__ void __launch_bounds__(256) pack_rows_kernel(int64_t n, const float2* __restrict__ xy,
                                                        const float* __restrict__ depth, const float* __restrict__ conic,
                                                        const float* __restrict__ comp, const float* __restrict__ opacity,
                                                        const float* __restrict__ rgb, const int32_t* __restrict__ radii,
                                                        const int32_t* __restrict__ scan, int32_t* __restrict__ row_index,
                                                        float* __restrict__ rows, int64_t* __restrict__ d_count) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int r = radii[i];
    const int64_t o = scan[i];
    if (i == n - 1) *d_count = o + (r > 0 ? 1 : 0);
    row_index[i] = (int32_t)o;
    if (r <= 0) return;
    float4* out = reinterpret_cast<float4*>(rows + o * B200GS_ROW_FLOATS);
    const float2 p = xy[i];
    out[0] = make_float4(p.x, p.y, depth[i], conic[3 * i]);
    out[1] = make_float4(conic[3 * i + 1], conic[3 * i + 2], comp ? comp[i] : 1.0f, opacity[i]);
    out[2] = make_float4(rgb[3 * i], rgb[3 * i + 1], rgb[3 * i + 2], __int_as_float(r));
}

}  // namespace

static size_t pack_scan_state_bytes(int64_t n) { return align_up((size_t)div_up64(n > 0 ? n : 1, 256) * 4 + 64, 256); }

static size_t pack_rows_workspace_bytes(int64_t n) { return pack_scan_state_bytes(n) + align_up((size_t)(n > 0 ? n : 1) * 4, 256); }

}  // namespace b200gs

using namespace b200gs;

extern "C" {

size_t b200gs_bin_count_workspace_bytes(int64_t n) { return n < 0 ? 0 : carve_a(nullptr, n).bytes; }

size_t b200gs_bin_sort_workspace_bytes(int64_t n, int64_t max_coarse, int32_t width, int32_t height) {
    if (n < 0 || max_coarse < 0 || width <= 0 || height <= 0) return 0;
    return carve_b(nullptr, n, max_coarse, width, height).bytes;
}

int b200gs_bin_count(int32_t mode, int32_t width, int32_t height, int64_t n, const float* xy, const float* depth,
                     const int32_t* radii, const float* cull_conic, const float* cull_opacity, void* workspace, size_t workspace_bytes,
                     int64_t* d_counts, int64_t* host_counts, int32_t sync_host, void* stream) {
    B200GS_CHECK_ARG(mode == B200GS_MODE_VANILLA || mode == B200GS_MODE_GSPLAT, "bad mode");
    B200GS_CHECK_ARG(width > 0 && height > 0 && n >= 0, "bad size");
    B200GS_CHECK_ARG(workspace && d_counts, "workspace/d_counts must not be NULL");
    B200GS_CHECK_ARG(n == 0 || (xy && depth && radii), "NULL pointer");
    B200GS_CHECK_ARG(n < (int64_t(1) << 31), "n >= 2^31");
    B200GS_CHECK_ARG((cull_conic == nullptr) == (cull_opacity == nullptr), "cull_conic and cull_opacity go together");
    return bin_count(mode, width, height, n, false, xy, depth, radii, cull_conic, cull_opacity, workspace, workspace_bytes, d_counts,
                     host_counts, sync_host, (cudaStream_t)stream);
}

int b200gs_bin_count_rows(int32_t mode, int32_t width, int32_t height, int64_t n, const float* rows, int32_t cull, void* workspace,
                          size_t workspace_bytes, int64_t* d_counts, int64_t* host_counts, int32_t sync_host, void* stream,
                          const int64_t* block_counts, int64_t block_rows) {
    B200GS_CHECK_ARG(mode == B200GS_MODE_VANILLA || mode == B200GS_MODE_GSPLAT, "bad mode");
    B200GS_CHECK_ARG(width > 0 && height > 0 && n >= 0 && n < (int64_t(1) << 31), "bad size");
    B200GS_CHECK_ARG(workspace && d_counts && (n == 0 || rows), "NULL pointer");
    B200GS_CHECK_ARG((reinterpret_cast<uintptr_t>(rows) & 15u) == 0, "rows must be 16-byte aligned");
    // the count kernel indexes the blocks in int (BinSrc::blk_rows)
    B200GS_CHECK_ARG(block_counts == nullptr || (block_rows > 0 && block_rows <= INT32_MAX), "block_rows must be 1..2^31-1 with block_counts");
    return bin_count(mode, width, height, n, true, rows + B200GS_ROW_XY, rows + B200GS_ROW_DEPTH, (const int32_t*)(rows + B200GS_ROW_RADIUS),
                     rows + B200GS_ROW_CONIC, rows + B200GS_ROW_OPACITY, workspace, workspace_bytes, d_counts, host_counts, sync_host,
                     (cudaStream_t)stream, block_counts, block_rows);
}

int b200gs_bin_sort(int32_t mode, int32_t width, int32_t height, int64_t n, int32_t cull, int64_t max_coarse, int64_t max_pairs,
                    int64_t* d_counts, const void* ws_a, void* ws_b, size_t ws_bytes, int32_t* sorted_ids, int32_t* tile_ranges,
                    int64_t* host_counts, int32_t sync_host, void* stream) {
    B200GS_CHECK_ARG(mode == B200GS_MODE_VANILLA || mode == B200GS_MODE_GSPLAT, "bad mode");
    B200GS_CHECK_ARG(width > 0 && height > 0 && n >= 0 && max_pairs >= 0 && max_coarse >= 0, "bad size");
    B200GS_CHECK_ARG(d_counts != nullptr, "d_counts must not be NULL");
    B200GS_CHECK_ARG(ws_a && ws_b && tile_ranges, "workspace/tile_ranges must not be NULL");
    B200GS_CHECK_ARG(n == 0 || max_coarse == 0 || sorted_ids, "NULL pointer");
    const cudaStream_t s = (cudaStream_t)stream;
    int grid_x, grid_y, cgrid_x, cgrid_y;
    cell_grid(width, height, grid_x, grid_y, cgrid_x, cgrid_y);
    const int n_tiles = grid_x * grid_y, n_cells = cgrid_x * cgrid_y;
    if (max_pairs >= (int64_t(1) << 30) || max_coarse >= (int64_t(1) << 30)) {
        set_error("bin_sort: capacity %lld / %lld exceeds 2^30", (long long)max_coarse, (long long)max_pairs);
        return B200GS_ENOSPACE;
    }
    if (n_cells > 65536) {
        set_error("bin_sort: %d coarse cells exceed 65536 (image too large)", n_cells);
        return B200GS_ENOSPACE;
    }
    if (max_coarse == 0 || n == 0) {   // nothing on screen (or nothing can be stored): empty lists; counts[2] stays 0
        B200GS_CUDA(cudaMemsetAsync(tile_ranges, 0, sizeof(int32_t) * 2 * (size_t)n_tiles, s));
        return publish_counts(d_counts, host_counts, sync_host, s);
    }
    const WorkspaceA A = carve_a(const_cast<void*>(ws_a), n);
    const WorkspaceB W = carve_b(ws_b, n, max_coarse, width, height);
    if (ws_bytes < W.bytes) {
        set_error("bin_sort: workspace too small (%zu < %zu)", ws_bytes, W.bytes);
        return B200GS_ENOSPACE;
    }
    const uint2* order = A.rec_a;
    const SplatRec* recs = A.recs;
    const int64_t* d_visible = d_counts + 3;
    const int64_t* d_coarse = d_counts + 1;

    // B: coarse entries with their tile masks in depth order; per-cell counts
    B200GS_CUDA(cudaMemsetAsync(W.cell_hist, 0, W.zero_bytes, s));
    const int passes = n_cells > sweep::RADIX ? 2 : 1;     // partition passes: one per byte of the cell id
    CellEntry* emit_dst = passes == 2 ? W.entries : W.entries_in;   // the partitioned entries end in W.entries
    const int pack = pack_ncells(n, width, height) ? 1 : 0;
    rank_offsets_kernel<<<(unsigned)W.scan_blocks, 256, 0, s>>>(d_visible, pack, order, recs, W.offsets, W.tickets, W.scan_state);
    B200GS_LAUNCH_CHECK();
    static constexpr decltype(&emit_cells_kernel<false>) emit[2] = {emit_cells_kernel<false>, emit_cells_kernel<true>};
    emit[mode == B200GS_MODE_GSPLAT]<<<(unsigned)W.blocks, 256, 0, s>>>(d_visible, pack, grid_x, grid_y, cgrid_x, cull, max_coarse, order, recs,
                                                                         W.offsets, emit_dst, n_cells, W.cell_hist);
    B200GS_LAUNCH_CHECK();
    cell_table_kernel<<<1, 1024, 0, s>>>(n_cells, W.cell_hist, W.cell_ranges, W.chunk_base, W.chunk_cell, W.digit_hist, n_tiles, W.tile_start);
    B200GS_LAUNCH_CHECK();
    // stable partition by cell (the entry carries its cell in .w)
    CellEntry* src_ent = emit_dst;
    CellEntry* dst_ent = passes == 2 ? W.entries_in : W.entries;
    for (int pass = 0; pass < passes; ++pass) {
        sweep::onesweep_pass_kernel<CellEntry, CELL_IPT><<<(unsigned)W.tiles, sweep::PASS_THREADS, 0, s>>>(
            src_ent, dst_ent, d_coarse, max_coarse, 8 * pass, W.digit_hist + pass * sweep::RADIX, W.lookback + (size_t)pass * W.tiles * sweep::RADIX,
            W.tickets + 1 + pass);
        B200GS_LAUNCH_CHECK();
        CellEntry* tmp = src_ent; src_ent = dst_ent; dst_ent = tmp;
    }

    // C: per-chunk tile counts;  D: chunk prefixes, tile starts / ranges / total;  E: ids in place
    const unsigned chunks = (unsigned)W.max_chunks;
    chunk_counts_kernel<<<chunks, CHUNK, 0, s>>>(n_cells, cgrid_x, grid_x, grid_y, W.cell_ranges, W.chunk_base, W.chunk_cell, W.entries, W.chunk_cnt,
                                                 W.tile_start);
    B200GS_LAUNCH_CHECK();
    chunk_prefix_kernel<<<(unsigned)n_cells + 1, 1024, 0, s>>>(n_cells, n_tiles, W.chunk_base, W.chunk_cnt, W.chunk_pre, W.tile_start, max_pairs,
                                                               (int2*)tile_ranges, d_counts);
    B200GS_LAUNCH_CHECK();
    scatter_ids_kernel<<<chunks, CHUNK, 0, s>>>(n_cells, cgrid_x, grid_x, grid_y, max_pairs, W.cell_ranges, W.chunk_base, W.chunk_cell, W.entries,
                                                W.chunk_pre, W.tile_start, sorted_ids);
    B200GS_LAUNCH_CHECK();
    return publish_counts(d_counts, host_counts, sync_host, s);
}

int b200gs_publish_i64(const int64_t* d_values, int64_t* host_values, int32_t n, void* stream) {
    B200GS_CHECK_ARG(d_values && host_values && n > 0, "bad argument");
    return publish_i64(d_values, host_values, n, (cudaStream_t)stream);
}

// ---- [n,12] row layout (the exchange format of the Gaussian-sharded renderer) -------------------------------------------
size_t b200gs_pack_rows_workspace_bytes(int64_t n) { return n < 0 ? 0 : pack_rows_workspace_bytes(n); }

int b200gs_pack_rows(int64_t n, const float* xy, const float* depth, const float* conic, const float* comp, const float* opacity,
                     const float* rgb, const int32_t* radii, void* ws, size_t workspace_bytes, int32_t* row_index, float* rows,
                     int64_t* d_count, void* stream) {
    B200GS_CHECK_ARG(n >= 0 && n < (int64_t(1) << 31), "bad n");
    B200GS_CHECK_ARG(d_count != nullptr, "d_count must not be NULL");
    B200GS_CHECK_ARG(n == 0 || (xy && depth && conic && opacity && rgb && radii && ws && row_index && rows), "NULL pointer");
    B200GS_CHECK_ARG(n == 0 || workspace_bytes >= pack_rows_workspace_bytes(n), "workspace too small");
    const cudaStream_t s = (cudaStream_t)stream;
    if (n == 0) {
        B200GS_CUDA(cudaMemsetAsync(d_count, 0, sizeof(int64_t), s));
        return B200GS_OK;
    }
    const size_t state_bytes = pack_scan_state_bytes(n);
    uint32_t* ticket = (uint32_t*)ws;               // [0]: ticket, [16..]: chained-scan state of the blocks
    uint32_t* state = ticket + 16;
    int32_t* scan = (int32_t*)((char*)ws + state_bytes);
    B200GS_CUDA(cudaMemsetAsync(ws, 0, state_bytes, s));
    visible_scan_kernel<<<(unsigned)div_up64(n, 256 * VS_ITEMS), 256, 0, s>>>(n, radii, scan, ticket, state);
    B200GS_LAUNCH_CHECK();
    pack_rows_kernel<<<(unsigned)div_up64(n, 256), 256, 0, s>>>(n, (const float2*)xy, depth, conic, comp, opacity, rgb, radii, scan, row_index,
                                                               rows, d_count);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

}  // extern "C"
