// distCUDA2 of simple-knn (the initialiser of the Gaussians' scales: internal/models/vanilla_gaussian.py:122-125 calls
// `simple_knn._C.distCUDA2(points)` once per run): for every point the MEAN of the squared distances to its 3 nearest neighbours.
// simple-knn@44f7642 orders the points along a Morton curve and prunes with bounding boxes; the result is the exact 3-NN mean.
// pytorch3d's knn_points (the similarity regulariser of internal/metrics/appearance_feature_similarity_regularization_metrics.py
// and SegAny's feature smoothing): for every query the K <= 32 nearest reference points, self included, in ascending order.
// Both run on one grid build: a uniform hash grid (about two points per cell) sized on the device from the bounding box, the points
// sorted by cell with the library's own onesweep radix passes, a dense first/last table per cell; then one thread per point or query
// searches growing shells of cells until its K-th best distance is no larger than the distance to the unsearched region.  Nothing is
// copied to the host: the radix pass count follows from the host-known cell capacity, and the kernels read the grid from the
// workspace.
#include <float.h>

#include "common.cuh"
#include "knn_grid.h"
#include "onesweep.cuh"

namespace b200gs {

namespace {

// clamped before the conversion, so an infinite or NaN offset (a non-finite point, an overflowing difference) lands in an edge cell
__device__ __forceinline__ int cell_coord(float v, float lo, float inv_cs, int g) { return (int)fminf(fmaxf((v - lo) * inv_cs, 0.f), (float)(g - 1)); }

// float -> uint32 with the same order (finite values), and back
__device__ __forceinline__ uint32_t ordered_key(float f) {
    const uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float from_ordered_key(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

// bounds[0..2] = ~key(min xyz), bounds[3..5] = key(max xyz) over the points whose three coordinates are finite: both maxima, so the
// zero-initialised workspace is the identity (and decodes to NaN bounds, which the sizing treats as empty, when no point is finite)
__global__ void __launch_bounds__(256) knn_bounds_kernel(int64_t n, const float* __restrict__ pts, uint32_t* __restrict__ bounds) {
    float lo[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, hi[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
    for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += int64_t(gridDim.x) * blockDim.x) {
        const float x = pts[3 * i], y = pts[3 * i + 1], z = pts[3 * i + 2];
        if (!(isfinite(x) && isfinite(y) && isfinite(z))) continue;
        lo[0] = fminf(lo[0], x); lo[1] = fminf(lo[1], y); lo[2] = fminf(lo[2], z);
        hi[0] = fmaxf(hi[0], x); hi[1] = fmaxf(hi[1], y); hi[2] = fmaxf(hi[2], z);
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        lo[a] = warp_reduce<Min>(lo[a]);
        hi[a] = warp_reduce<Max>(hi[a]);
    }
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            atomicMax(bounds + a, ~ordered_key(lo[a]));
            atomicMax(bounds + 3 + a, ordered_key(hi[a]));
        }
    }
}

// size_knn_grid (knn_grid.h) in one thread
__global__ void knn_grid_kernel(int64_t n, const uint32_t* __restrict__ bounds, int64_t max_cells, KnnGrid* __restrict__ grid) {
    float lo[3], hi[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        lo[a] = from_ordered_key(~bounds[a]);
        hi[a] = from_ordered_key(bounds[3 + a]);
    }
    *grid = size_knn_grid(lo, hi, n, max_cells);
}

__global__ void __launch_bounds__(256) knn_keys_kernel(int64_t n, const float* __restrict__ pts, const KnnGrid* __restrict__ grid, uint2* __restrict__ rec) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const KnnGrid g = *grid;
    const int cx = cell_coord(pts[3 * i], g.lox, g.inv_cs, g.gx), cy = cell_coord(pts[3 * i + 1], g.loy, g.inv_cs, g.gy),
              cz = cell_coord(pts[3 * i + 2], g.loz, g.inv_cs, g.gz);
    rec[i] = make_uint2((uint32_t)((cz * g.gy + cy) * g.gx + cx), (uint32_t)i);
}

// sorted position -> point (x, y, z, original index) and the first / last position of every cell
__global__ void __launch_bounds__(256) knn_gather_kernel(int64_t n, const float* __restrict__ pts, const uint2* __restrict__ rec, float4* __restrict__ sorted,
                                                         int* __restrict__ cell_lo, int* __restrict__ cell_hi) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint2 r = rec[i];
    sorted[i] = make_float4(pts[3 * (int64_t)r.y], pts[3 * (int64_t)r.y + 1], pts[3 * (int64_t)r.y + 2], __int_as_float((int)r.y));
    if (i == 0 || rec[i - 1].x != r.x) cell_lo[r.x] = (int)i;
    if (i == n - 1 || rec[i + 1].x != r.x) cell_hi[r.x] = (int)i + 1;
}

__device__ __forceinline__ void knn_insert(float d, float& b0, float& b1, float& b2) {
    if (d < b2) {
        if (d < b1) {
            b2 = b1;
            if (d < b0) { b1 = b0; b0 = d; } else b1 = d;
        } else b2 = d;
    }
}

__global__ void __launch_bounds__(128) knn_search_kernel(int64_t n, const float4* __restrict__ sorted, const int* __restrict__ cell_lo,
                                                         const int* __restrict__ cell_hi, const KnnGrid* __restrict__ grid, float* __restrict__ out) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const KnnGrid g = *grid;
    const float4 p = sorted[i];
    const int cx = cell_coord(p.x, g.lox, g.inv_cs, g.gx), cy = cell_coord(p.y, g.loy, g.inv_cs, g.gy), cz = cell_coord(p.z, g.loz, g.inv_cs, g.gz);
    float b0 = FLT_MAX, b1 = FLT_MAX, b2 = FLT_MAX;
    const int rmax = max(g.gx, max(g.gy, g.gz));
    for (int r = 0; r <= rmax; ++r) {
        for (int dz = -r; dz <= r; ++dz) {
            const int z = cz + dz;
            if (z < 0 || z >= g.gz) continue;
            for (int dy = -r; dy <= r; ++dy) {
                const int y = cy + dy;
                if (y < 0 || y >= g.gy) continue;
                const bool face = (abs(dz) == r) || (abs(dy) == r);
                for (int dx = -r; dx <= r; dx += (face ? 1 : max(1, 2 * r))) {   // only the shell at Chebyshev distance r
                    const int x = cx + dx;
                    if (x < 0 || x >= g.gx) continue;
                    const int c = (z * g.gy + y) * g.gx + x;
                    const int lo = cell_lo[c], hi = cell_hi[c];
                    for (int j = lo; j < hi; ++j) {
                        if (j == (int)i) continue;
                        const float4 q = sorted[j];
                        const float ex = q.x - p.x, ey = q.y - p.y, ez = q.z - p.z;
                        knn_insert(ex * ex + ey * ey + ez * ez, b0, b1, b2);
                    }
                }
            }
        }
        // everything outside the searched cube is at least r cells away from this point's own cell, i.e. >= r * cs from the point
        const float reach = float(r) * g.cs;
        if (b2 <= reach * reach) break;
    }
    // fewer than 3 other points in the whole set: the missing distances count as 0, i.e. the sum of those there are over 3, and 0
    // for a single point (simple-knn leaves such inputs undefined)
    float sum = 0.f;
    int cnt = 0;
    if (b0 < FLT_MAX) { sum += b0; ++cnt; }
    if (b1 < FLT_MAX) { sum += b1; ++cnt; }
    if (b2 < FLT_MAX) { sum += b2; ++cnt; }
    out[__float_as_int(p.w)] = cnt ? sum / 3.0f : 0.f;
}

// histograms of the four key bytes of the uint2 records: the digit counts of all the radix passes at once
constexpr int HIST_THREADS = 256;
constexpr int SORT_IPT = 8;

__global__ void __launch_bounds__(HIST_THREADS) hist4_kernel(const uint2* __restrict__ recs, const int64_t* __restrict__ d_n, int64_t cap,
                                                             uint32_t* __restrict__ hist /*[4][RADIX]*/) {
    using sweep::RADIX;
    __shared__ uint32_t s_h[4][RADIX];
    const int64_t n = d_n ? min(cap, *d_n) : cap;
    for (int i = threadIdx.x; i < 4 * RADIX; i += HIST_THREADS) (&s_h[0][0])[i] = 0;
    __syncthreads();
    for (int64_t i = int64_t(blockIdx.x) * HIST_THREADS + threadIdx.x; i < n; i += int64_t(gridDim.x) * HIST_THREADS) {
        const uint32_t k = recs[i].x;
        atomicAdd(&s_h[0][k & 255u], 1u);
        atomicAdd(&s_h[1][(k >> 8) & 255u], 1u);
        atomicAdd(&s_h[2][(k >> 16) & 255u], 1u);
        atomicAdd(&s_h[3][k >> 24], 1u);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 4 * RADIX; i += HIST_THREADS) {
        const uint32_t c = (&s_h[0][0])[i];
        if (c) atomicAdd(hist + i, c);
    }
}

// ---- the K nearest reference points of arbitrary queries --------------------------------------------------------------
// Insert (d, j) into the ascending list of the KC best: a fixed sequence of selects over the whole list, so it stays in registers.
// Strict comparisons keep an earlier-inserted point ahead of a later one at the same distance.
template <int KC>
__device__ __forceinline__ void list_insert(float d, int j, float (&bd)[KC], int (&bi)[KC]) {
#pragma unroll
    for (int t = KC - 1; t > 0; --t) {
        const bool shift = d < bd[t - 1], here = !shift && d < bd[t];
        bi[t] = shift ? bi[t - 1] : (here ? j : bi[t]);
        bd[t] = shift ? bd[t - 1] : (here ? d : bd[t]);
    }
    const bool first = d < bd[0];
    bi[0] = first ? j : bi[0];
    bd[0] = first ? d : bd[0];
}

// One thread per query: the list holds the KC >= k best (KC a power of two), the search stops once the k-th best is no larger than
// the distance to every unsearched cell.  A query outside the grid's box is clamped to its edge cell; every cell at Chebyshev index
// distance > r from that cell still lies more than r cells away from the query along some axis, so the bound holds there too.  The
// bound is shrunk by 2^-10 of a cell, which covers the rounding of the cell coordinates.
template <int KC>
__global__ void __launch_bounds__(128) knn_query_kernel(int64_t s, const float* __restrict__ queries, int k, const float4* __restrict__ sorted,
                                                        const int* __restrict__ cell_lo, const int* __restrict__ cell_hi,
                                                        const KnnGrid* __restrict__ grid, const float* __restrict__ points,
                                                        float* __restrict__ dists, int64_t* __restrict__ idx) {
    const int64_t q = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (q >= s) return;
    const KnnGrid g = *grid;
    const float px = queries[3 * q], py = queries[3 * q + 1], pz = queries[3 * q + 2];
    const int cx = cell_coord(px, g.lox, g.inv_cs, g.gx), cy = cell_coord(py, g.loy, g.inv_cs, g.gy), cz = cell_coord(pz, g.loz, g.inv_cs, g.gz);
    float bd[KC];
    int bi[KC];
#pragma unroll
    for (int t = 0; t < KC; ++t) { bd[t] = FLT_MAX; bi[t] = -1; }
    const int rmax = max(g.gx, max(g.gy, g.gz));
    for (int r = 0; r <= rmax; ++r) {
        for (int dz = -r; dz <= r; ++dz) {
            const int z = cz + dz;
            if (z < 0 || z >= g.gz) continue;
            for (int dy = -r; dy <= r; ++dy) {
                const int y = cy + dy;
                if (y < 0 || y >= g.gy) continue;
                const bool face = (abs(dz) == r) || (abs(dy) == r);
                for (int dx = -r; dx <= r; dx += (face ? 1 : max(1, 2 * r))) {
                    const int x = cx + dx;
                    if (x < 0 || x >= g.gx) continue;
                    const int c = (z * g.gy + y) * g.gx + x;
                    const int lo = cell_lo[c], hi = cell_hi[c];
                    for (int j = lo; j < hi; ++j) {
                        const float4 p = sorted[j];
                        const float ex = p.x - px, ey = p.y - py, ez = p.z - pz;
                        const float d = ex * ex + ey * ey + ez * ez;
                        if (d < bd[KC - 1]) list_insert<KC>(d, __float_as_int(p.w), bd, bi);
                    }
                }
            }
        }
        float kth = bd[0];
#pragma unroll
        for (int t = 1; t < KC; ++t) kth = (t == k - 1) ? bd[t] : kth;
        const float reach = float(r) * g.cs * (1.f - 1.f / 1024.f);
        if (kth <= reach * reach) break;
    }
    // Fewer than k points at a finite distance below FLT_MAX (a query with a NaN or infinite coordinate, or non-finite reference
    // points): the empty slots take the lowest indices not in the list, as pytorch3d keeps its first candidates when no distance
    // compares smaller, with their distances as computed (NaN or inf).  Every index written is in [0, n).
    bool short_list = false;
#pragma unroll
    for (int t = 0; t < KC; ++t) short_list = short_list || (t < k && bi[t] < 0);
    if (short_list) {
        int next = 0;
#pragma unroll
        for (int t = 0; t < KC; ++t) {
            if (t < k && bi[t] < 0) {
                for (bool taken = true; taken;) {
                    taken = false;
#pragma unroll
                    for (int u = 0; u < KC; ++u) taken = taken || bi[u] == next;
                    if (taken) ++next;
                }
                const float ex = points[3 * (int64_t)next] - px, ey = points[3 * (int64_t)next + 1] - py, ez = points[3 * (int64_t)next + 2] - pz;
                bi[t] = next++;
                bd[t] = ex * ex + ey * ey + ez * ez;
            }
        }
    }
#pragma unroll
    for (int t = 0; t < KC; ++t) {
        if (t < k) {
            dists[q * k + t] = bd[t];
            idx[q * k + t] = bi[t];
        }
    }
}

struct KnnLayout {
    size_t grid, sorted, rec_a, rec_b, zero, bounds, sort_scratch, cell_lo, cell_hi, zero_bytes, total;
    int64_t max_cells;
};

KnnLayout knn_layout(int64_t n) {
    KnnLayout L{};
    size_t off = 0;
    auto take = [&off](size_t bytes) { size_t o = off; off = align_up(off + bytes, 256); return o; };
    const size_t nn = (size_t)(n > 0 ? n : 1);
    L.max_cells = (int64_t)(4 * nn + 64);
    L.grid = take(sizeof(KnnGrid));
    L.sorted = take(nn * 16);
    L.rec_a = take(nn * 8);
    L.rec_b = take(nn * 8);
    L.zero = off;                                    // one memset clears the bounds, the sort's counters and the cell table
    L.bounds = take(6 * 4);
    L.sort_scratch = take(record_sort_scratch_bytes((int64_t)nn));
    L.cell_hi = take((size_t)L.max_cells * 4);      // empty cells have lo = hi = 0
    L.cell_lo = take((size_t)L.max_cells * 4);
    L.zero_bytes = off - L.zero;
    L.total = off;
    return L;
}

// bounds -> grid -> cell keys -> sort by cell -> sorted points and the cell table
int build_grid(int64_t n, const float* points, const KnnLayout& L, char* w, cudaStream_t s) {
    uint32_t* bounds = (uint32_t*)(w + L.bounds);
    KnnGrid* grid = (KnnGrid*)(w + L.grid);
    uint2* rec_a = (uint2*)(w + L.rec_a);
    uint2* rec_b = (uint2*)(w + L.rec_b);
    B200GS_CUDA(cudaMemsetAsync(w + L.zero, 0, L.zero_bytes, s));
    knn_bounds_kernel<<<(unsigned)min((int64_t)1184, div_up64(n, 256)), 256, 0, s>>>(n, points, bounds);
    B200GS_LAUNCH_CHECK();
    knn_grid_kernel<<<1, 1, 0, s>>>(n, bounds, L.max_cells, grid);
    B200GS_LAUNCH_CHECK();
    const unsigned blocks = (unsigned)div_up64(n, 256);
    knn_keys_kernel<<<blocks, 256, 0, s>>>(n, points, grid, rec_a);
    B200GS_LAUNCH_CHECK();
    const uint2* sorted_rec = nullptr;
    if (int rc = launch_record_sort(n, record_key_bits(L.max_cells - 1), rec_a, rec_b, w + L.sort_scratch, s, &sorted_rec)) return rc;
    knn_gather_kernel<<<blocks, 256, 0, s>>>(n, points, sorted_rec, (float4*)(w + L.sorted), (int*)(w + L.cell_lo), (int*)(w + L.cell_hi));
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

int check_knn_workspace(int64_t n, size_t ws_bytes) {
    const size_t need = knn_layout(n).total;
    if (ws_bytes < need) {
        set_error("knn: workspace too small (%zu < %zu)", ws_bytes, need);
        return B200GS_ENOSPACE;
    }
    if (n >= (int64_t(1) << 30)) {
        set_error("knn: %lld points exceed 2^30", (long long)n);
        return B200GS_ENOSPACE;
    }
    return B200GS_OK;
}

size_t sort_counters_bytes() { return align_up(4 * sweep::RADIX * 4 + 16 * 4, 256); }

}  // namespace

int record_key_bits(int64_t max_key) {
    int bits = 1;
    while (bits < 32 && (int64_t(1) << bits) <= max_key) ++bits;
    return bits;
}

size_t record_sort_scratch_bytes(int64_t n) {
    const int64_t tiles = div_up64(n > 0 ? n : 1, sweep::PASS_THREADS * SORT_IPT);
    return sort_counters_bytes() + (size_t)4 * tiles * sweep::RADIX * 4;
}

int launch_record_sort(int64_t n, int bits, uint2* a, uint2* b, void* scratch, cudaStream_t s, const uint2** out) {
    *out = a;
    if (n == 0) return B200GS_OK;
    const int64_t tiles = div_up64(n, sweep::PASS_THREADS * SORT_IPT);
    uint32_t* hist = (uint32_t*)scratch;
    uint32_t* tickets = hist + 4 * sweep::RADIX;
    uint32_t* lookback = (uint32_t*)((char*)scratch + sort_counters_bytes());
    hist4_kernel<<<(unsigned)min((int64_t)592, div_up64(n, 256)), HIST_THREADS, 0, s>>>(a, nullptr, n, hist);
    B200GS_LAUNCH_CHECK();
    uint2* src = a;
    uint2* dst = b;
    for (int pass = 0; pass < (bits + 7) / 8; ++pass) {
        sweep::onesweep_pass_kernel<uint2, SORT_IPT><<<(unsigned)tiles, sweep::PASS_THREADS, 0, s>>>(src, dst, nullptr, n, 8 * pass, hist + pass * sweep::RADIX,
                                                                                          lookback + (size_t)pass * tiles * sweep::RADIX, tickets + pass);
        B200GS_LAUNCH_CHECK();
        uint2* t = src; src = dst; dst = t;
    }
    *out = src;
    return B200GS_OK;
}

}  // namespace b200gs

using namespace b200gs;

extern "C" {

// both entry points share the workspace layout knn_layout
size_t b200gs_knn_workspace_bytes(int64_t n) { return n < 0 ? 0 : knn_layout(n).total; }

int b200gs_knn_mean_dist2(int64_t n, const float* points, float* mean_dist2, void* workspace, size_t workspace_bytes, void* stream) {
    B200GS_CHECK_ARG(n >= 0, "n < 0");
    B200GS_CHECK_ARG(n == 0 || (points && mean_dist2 && workspace), "NULL pointer");
    if (n == 0) return B200GS_OK;
    if (int rc = check_knn_workspace(n, workspace_bytes)) return rc;
    const cudaStream_t s = (cudaStream_t)stream;
    const KnnLayout L = knn_layout(n);
    char* w = (char*)workspace;
    if (int rc = build_grid(n, points, L, w, s)) return rc;
    knn_search_kernel<<<(unsigned)div_up64(n, 128), 128, 0, s>>>(n, (const float4*)(w + L.sorted), (const int*)(w + L.cell_lo),
                                                                (const int*)(w + L.cell_hi), (const KnnGrid*)(w + L.grid), mean_dist2);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

int b200gs_knn_points(int64_t s_q, const float* queries, int64_t n, const float* points, int32_t k, float* dists, int64_t* idx,
                      void* workspace, size_t workspace_bytes, void* stream) {
    B200GS_CHECK_ARG(s_q >= 0 && n >= 0, "negative size");
    B200GS_CHECK_ARG(k >= 1 && k <= 32, "K must be 1..32");
    B200GS_CHECK_ARG(k <= n, "K exceeds the number of reference points");
    B200GS_CHECK_ARG(points && workspace, "NULL pointer");
    B200GS_CHECK_ARG(s_q == 0 || (queries && dists && idx), "NULL pointer");
    if (int rc = check_knn_workspace(n, workspace_bytes)) return rc;
    if (s_q == 0) return B200GS_OK;
    const cudaStream_t s = (cudaStream_t)stream;
    const KnnLayout L = knn_layout(n);
    char* w = (char*)workspace;
    if (int rc = build_grid(n, points, L, w, s)) return rc;
    const unsigned blocks = (unsigned)div_up64(s_q, 128);
    const float4* sorted = (const float4*)(w + L.sorted);
    const int* lo = (const int*)(w + L.cell_lo);
    const int* hi = (const int*)(w + L.cell_hi);
    const KnnGrid* grid = (const KnnGrid*)(w + L.grid);
    if (k <= 1) knn_query_kernel<1><<<blocks, 128, 0, s>>>(s_q, queries, k, sorted, lo, hi, grid, points, dists, idx);
    else if (k <= 2) knn_query_kernel<2><<<blocks, 128, 0, s>>>(s_q, queries, k, sorted, lo, hi, grid, points, dists, idx);
    else if (k <= 4) knn_query_kernel<4><<<blocks, 128, 0, s>>>(s_q, queries, k, sorted, lo, hi, grid, points, dists, idx);
    else if (k <= 8) knn_query_kernel<8><<<blocks, 128, 0, s>>>(s_q, queries, k, sorted, lo, hi, grid, points, dists, idx);
    else if (k <= 16) knn_query_kernel<16><<<blocks, 128, 0, s>>>(s_q, queries, k, sorted, lo, hi, grid, points, dists, idx);
    else knn_query_kernel<32><<<blocks, 128, 0, s>>>(s_q, queries, k, sorted, lo, hi, grid, points, dists, idx);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

}  // extern "C"
