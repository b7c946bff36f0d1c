// distCUDA2 of simple-knn (the initialiser of the Gaussians' scales: internal/models/vanilla_gaussian.py:122-125 calls
// `simple_knn._C.distCUDA2(points)` once per run): for every point the MEAN of the squared distances to its 3 nearest neighbours.
// simple-knn@44f7642 orders the points along a Morton curve and prunes with bounding boxes; the result is the exact 3-NN mean.
// Here: a uniform hash grid (about two points per cell), the points sorted by cell with the library's own onesweep radix
// passes, a dense first/last table per cell, and one thread per point that searches growing shells of cells until the third
// best distance is no larger than the distance to the unsearched region — also the exact 3-NN (ties aside).
#include <float.h>

#include "common.cuh"
#include "onesweep.cuh"

namespace b200gs {

namespace {

struct KnnGrid {
    float lox, loy, loz, cs, inv_cs;
    int gx, gy, gz;
};

__device__ __forceinline__ int cell_coord(float v, float lo, float inv_cs, int g) { return min(g - 1, max(0, (int)((v - lo) * inv_cs))); }

__global__ void __launch_bounds__(256) knn_bounds_kernel(int64_t n, const float* __restrict__ pts, float* __restrict__ bounds /*[6]: min xyz, max xyz*/) {
    float lo[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, hi[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
    for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += int64_t(gridDim.x) * blockDim.x)
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const float v = pts[3 * i + a];
            lo[a] = fminf(lo[a], v);
            hi[a] = fmaxf(hi[a], v);
        }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            lo[a] = fminf(lo[a], __shfl_xor_sync(0xffffffffu, lo[a], o));
            hi[a] = fmaxf(hi[a], __shfl_xor_sync(0xffffffffu, hi[a], o));
        }
    }
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {   // float atomics through the order-preserving int view (all values finite)
            atomicMin(reinterpret_cast<int*>(bounds + a), lo[a] >= 0.f ? __float_as_int(lo[a]) : (int)(0x80000000u - (unsigned)__float_as_int(lo[a])));
            atomicMax(reinterpret_cast<int*>(bounds + 3 + a), hi[a] >= 0.f ? __float_as_int(hi[a]) : (int)(0x80000000u - (unsigned)__float_as_int(hi[a])));
        }
    }
}

__global__ void __launch_bounds__(256) knn_keys_kernel(int64_t n, const float* __restrict__ pts, const KnnGrid g, uint2* __restrict__ rec) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
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
                                                         const int* __restrict__ cell_hi, const KnnGrid g, float* __restrict__ out) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
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

struct KnnLayout {
    size_t bounds, rec_a, rec_b, sorted, zero, zero_bytes, hist, tickets, lookback, cell_lo, cell_hi, total;
    int64_t tiles, max_cells;
};

constexpr int KNN_IPT = 8;

KnnLayout knn_layout(int64_t n) {
    KnnLayout L{};
    size_t off = 0;
    auto take = [&off](size_t bytes) { size_t o = off; off = align_up(off + bytes, 256); return o; };
    const size_t nn = (size_t)(n > 0 ? n : 1);
    L.tiles = div_up64((int64_t)nn, sweep::PASS_THREADS * KNN_IPT);
    L.max_cells = (int64_t)(4 * nn + 64);
    L.bounds = take(6 * 4);
    L.rec_a = take(nn * 8);
    L.rec_b = take(nn * 8);
    L.sorted = take(nn * 16);
    L.zero = take(0);
    L.hist = take(4 * sweep::RADIX * 4);
    L.tickets = take(16 * 4);
    L.lookback = take((size_t)4 * L.tiles * sweep::RADIX * 4);
    L.cell_hi = take((size_t)L.max_cells * 4);      // zero-initialised with the region: empty cells have lo = hi = 0
    L.cell_lo = take((size_t)L.max_cells * 4);
    L.zero_bytes = off - L.zero;
    L.total = off;
    return L;
}

}  // namespace

size_t knn_workspace_bytes(int64_t n) { return knn_layout(n).total; }

int launch_knn_mean_dist2(int64_t n, const float* points, float* out, void* ws, size_t ws_bytes, cudaStream_t s) {
    if (n == 0) return B200GS_OK;
    const KnnLayout L = knn_layout(n);
    if (ws_bytes < L.total) {
        set_error("knn: workspace too small (%zu < %zu)", ws_bytes, L.total);
        return B200GS_ENOSPACE;
    }
    if (n >= (int64_t(1) << 30)) {
        set_error("knn: %lld points exceed 2^30", (long long)n);
        return B200GS_ENOSPACE;
    }
    char* w = (char*)ws;
    float* bounds = (float*)(w + L.bounds);
    // bounding box (the one host round trip of this init-only routine: the grid is sized on the host)
    const int init[6] = {0x7f7fffff, 0x7f7fffff, 0x7f7fffff, (int)0x80800001u, (int)0x80800001u, (int)0x80800001u};   // +FLT_MAX / -FLT_MAX in the ordered int view
    B200GS_CUDA(cudaMemcpyAsync(bounds, init, sizeof(init), cudaMemcpyHostToDevice, s));
    knn_bounds_kernel<<<(unsigned)min((int64_t)1184, div_up64(n, 256)), 256, 0, s>>>(n, points, bounds);
    B200GS_LAUNCH_CHECK();
    int hb[6];
    B200GS_CUDA(cudaMemcpyAsync(hb, bounds, sizeof(hb), cudaMemcpyDeviceToHost, s));
    B200GS_CUDA(cudaStreamSynchronize(s));
    float b[6];
    for (int a = 0; a < 6; ++a) {
        const int v = hb[a];
        const unsigned u = v >= 0 ? (unsigned)v : (0x80000000u - (unsigned)v);
        memcpy(&b[a], &u, 4);
    }
    const float ex = fmaxf(b[3] - b[0], 0.f), ey = fmaxf(b[4] - b[1], 0.f), ez = fmaxf(b[5] - b[2], 0.f);
    const float emax = fmaxf(ex, fmaxf(ey, ez));
    KnnGrid g{};
    g.lox = b[0]; g.loy = b[1]; g.loz = b[2];
    // about two points per OCCUPIED-volume cell; flat or linear point sets fall back to their largest extent
    double vol = (double)fmaxf(ex, 1e-3f * emax) * fmaxf(ey, 1e-3f * emax) * fmaxf(ez, 1e-3f * emax);
    float cs = emax > 0.f ? (float)cbrt(vol / (0.5 * (double)n)) : 1.0f;
    if (!(cs > 0.f)) cs = 1.0f;
    for (;;) {   // at most 1024 cells per axis and max_cells in total
        g.gx = (int)fminf(1024.f, floorf(ex / cs) + 1.f);
        g.gy = (int)fminf(1024.f, floorf(ey / cs) + 1.f);
        g.gz = (int)fminf(1024.f, floorf(ez / cs) + 1.f);
        if ((int64_t)g.gx * g.gy * g.gz <= L.max_cells && ex / cs < 1024.f && ey / cs < 1024.f && ez / cs < 1024.f) break;
        cs *= 1.26f;
    }
    g.cs = cs;
    g.inv_cs = 1.0f / cs;
    const int64_t n_cells = (int64_t)g.gx * g.gy * g.gz;

    uint2* rec_a = (uint2*)(w + L.rec_a);
    uint2* rec_b = (uint2*)(w + L.rec_b);
    float4* sorted = (float4*)(w + L.sorted);
    uint32_t* hist = (uint32_t*)(w + L.hist);
    uint32_t* tickets = (uint32_t*)(w + L.tickets);
    uint32_t* lookback = (uint32_t*)(w + L.lookback);
    int* cell_lo = (int*)(w + L.cell_lo);
    int* cell_hi = (int*)(w + L.cell_hi);
    B200GS_CUDA(cudaMemsetAsync(w + L.zero, 0, L.zero_bytes, s));
    const unsigned blocks = (unsigned)div_up64(n, 256);
    knn_keys_kernel<<<blocks, 256, 0, s>>>(n, points, g, rec_a);
    B200GS_LAUNCH_CHECK();
    hist4_kernel<<<(unsigned)min((int64_t)592, (int64_t)blocks), HIST_THREADS, 0, s>>>(rec_a, nullptr, n, hist);
    B200GS_LAUNCH_CHECK();
    int bits = 1;
    while ((int64_t(1) << bits) < n_cells) ++bits;
    const int passes = (bits + 7) / 8;
    uint2* src = rec_a;
    uint2* dst = rec_b;
    for (int pass = 0; pass < passes; ++pass) {
        sweep::onesweep_pass_kernel<uint2, KNN_IPT><<<(unsigned)L.tiles, sweep::PASS_THREADS, 0, s>>>(src, dst, nullptr, n, 8 * pass, hist + pass * sweep::RADIX,
                                                                                            lookback + (size_t)pass * L.tiles * sweep::RADIX, tickets + pass);
        B200GS_LAUNCH_CHECK();
        uint2* t = src; src = dst; dst = t;
    }
    knn_gather_kernel<<<blocks, 256, 0, s>>>(n, points, src, sorted, cell_lo, cell_hi);
    B200GS_LAUNCH_CHECK();
    knn_search_kernel<<<(unsigned)div_up64(n, 128), 128, 0, s>>>(n, sorted, cell_lo, cell_hi, g, out);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

}  // namespace b200gs
