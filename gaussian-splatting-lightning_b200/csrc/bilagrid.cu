// Bilateral-grid colour correction (BilaRF: Wang et al., "Bilateral Guided Radiance Field Processing", 2024), the per-image affine
// colour transform of internal/output_processors/bilagrid.py that runs between the render and the loss on every training step.
// A grid G = grids[g] (12, L, Hg, Wg) holds a 3x4 affine matrix A per cell; a pixel with coordinates (x, y) in [0,1] and colour
// rgb reads A by trilinear interpolation at
//     ix = x (Wg - 1),  iy = y (Hg - 1),  iz = gray (L - 1),  gray = 0.299 r + 0.587 g + 0.114 b
// (the align_corners=True unnormalisation of grid_sample, written in its op order), each clipped to [0, size - 1] (border padding),
// and outputs out_i = sum_j A_ij rgb_j + A_i3.  Gradients follow torch's grid_sample: a clipped coordinate, including one landing
// exactly on a bound, passes no gradient (so black pixels, gray = 0, have none through the guidance).
//   * slice_fwd: one thread per pixel; rgb / out are addressed through element strides, so a permuted CHW render is read and written
//     in place.  The grid index is read on the device; an index outside [0, n_grids) makes the row NaN and reads no grid.
//   * slice_bwd: v_rgb per pixel; v_grids summed in shared memory over the box of cells the CTA's pixels touch (all L levels x 12
//     channels), after a warp reduction over the lanes that share a lower corner, and flushed once per CTA.  A CTA whose box does
//     not fit BOX_CAP (scattered xy) adds each pixel's 96 terms to global memory instead.
//   * tv_fwd / tv_bwd: total_variation_loss, per-CTA partial sums (summed by the caller in a fixed order) and the dense gradient.
#include "common.cuh"

namespace b200gs {

namespace {

constexpr int BT = 16;            // pixel tile edge of the slice kernels
constexpr int BOX_CAP = 4096;     // floats of the backward's shared grid-gradient box (16 KiB: 42 cells x 8 levels x 12)
constexpr int TV_THREADS = 256;
constexpr float GW0 = 0.299f, GW1 = 0.587f, GW2 = 0.114f;

// grid_sample's unnormalise + border clip of one coordinate in [-1, 1]; *g = d(clipped)/d(coord): 0 on or outside a bound, as
// torch's clip_coordinates_set_grad; a NaN coordinate clips to 0
__device__ __forceinline__ float clip_coord(float coord, int size, float* g) {
    const float i = ((coord + 1.f) / 2.f) * float(size - 1);
    const float hi = float(size - 1);
    *g = (i > 0.f && i < hi) ? 0.5f * hi : 0.f;
    return fminf(fmaxf(i, 0.f), hi);
}

struct Sample {
    int x0, y0, z0;       // lower corner, in range
    int dx, dy, dz;       // 1, or 0 where the upper corner lies outside the grid (its weight is then 0)
    float w[8];           // trilinear weights, corner k = (kz << 2) | (ky << 1) | kx
    float dgray;          // d iz / d gray (0 where iz is clipped)
};

__device__ __forceinline__ Sample make_sample(float x, float y, float r, float g, float b, int L, int gh, int gw) {
    Sample s;
    float unused, gz;
    const float ix = clip_coord((x - 0.5f) * 2.f, gw, &unused);
    const float iy = clip_coord((y - 0.5f) * 2.f, gh, &unused);
    const float gray = fmaf(b, GW2, fmaf(g, GW1, r * GW0));
    const float iz = clip_coord(gray * 2.f - 1.f, L, &gz);
    s.dgray = 2.f * gz;           // d iz / d gray = L - 1 inside the grid
    s.x0 = int(floorf(ix)); s.y0 = int(floorf(iy)); s.z0 = int(floorf(iz));
    s.dx = s.x0 + 1 < gw; s.dy = s.y0 + 1 < gh; s.dz = s.z0 + 1 < L;
    const float fx = ix - float(s.x0), fy = iy - float(s.y0), fz = iz - float(s.z0);
#pragma unroll
    for (int k = 0; k < 8; ++k)
        s.w[k] = ((k & 1) ? fx : 1.f - fx) * ((k & 2) ? fy : 1.f - fy) * ((k & 4) ? fz : 1.f - fz);
    return s;
}

__device__ __forceinline__ int64_t corner_offset(const Sample& s, int k, int gh, int gw) {
    return (int64_t(s.z0 + ((k >> 2) & 1) * s.dz) * gh + s.y0 + ((k >> 1) & 1) * s.dy) * gw + s.x0 + (k & 1) * s.dx;
}

// A (12 channels) and, when dA != nullptr, dA/diz
__device__ __forceinline__ void interpolate(const float* __restrict__ G, int64_t plane, const Sample& s, int gh, int gw, float* A,
                                            float* dA) {
    int64_t off[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) off[k] = corner_offset(s, k, gh, gw);
    const float wxy[4] = {s.w[0] + s.w[4], s.w[1] + s.w[5], s.w[2] + s.w[6], s.w[3] + s.w[7]};   // weights summed over z
#pragma unroll
    for (int c = 0; c < 12; ++c) {
        const float* Gc = G + c * plane;
        float a = 0.f, d = 0.f;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const float v = __ldg(Gc + off[k]);
            a = fmaf(s.w[k], v, a);
            if (dA) d = fmaf((k & 4) ? wxy[k & 3] : -wxy[k & 3], v, d);
        }
        A[c] = a;
        if (dA) dA[c] = d;
    }
}

__device__ __forceinline__ int64_t grid_of(const int64_t* __restrict__ grid_idx, int n_idx, int b) {
    return __ldg(grid_idx + (n_idx == 1 ? 0 : b));
}

__global__ void __launch_bounds__(BT * BT) slice_fwd_kernel(int n_grids, int L, int gh, int gw, const float* __restrict__ grids,
                                                            int height, int width, const float* __restrict__ xy,
                                                            const float* __restrict__ rgb, int64_t sb, int64_t sy, int64_t sx,
                                                            int64_t sc, const int64_t* __restrict__ grid_idx, int n_idx,
                                                            float* __restrict__ out) {
    const int x = blockIdx.x * BT + threadIdx.x, y = blockIdx.y * BT + threadIdx.y, b = blockIdx.z;
    if (x >= width || y >= height) return;
    const int64_t g = grid_of(grid_idx, n_idx, b);
    const int64_t p = sb * b + sy * y + sx * x;
    if (g < 0 || g >= n_grids) {
        out[p] = out[p + sc] = out[p + 2 * sc] = __int_as_float(0x7fffffff);
        return;
    }
    const float r0 = __ldg(rgb + p), r1 = __ldg(rgb + p + sc), r2 = __ldg(rgb + p + 2 * sc);
    const int64_t q = (int64_t(b) * height + y) * width + x;
    const Sample s = make_sample(__ldg(xy + 2 * q), __ldg(xy + 2 * q + 1), r0, r1, r2, L, gh, gw);
    const int64_t plane = int64_t(L) * gh * gw;
    float A[12];
    interpolate(grids + g * 12 * plane, plane, s, gh, gw, A, nullptr);
#pragma unroll
    for (int i = 0; i < 3; ++i) out[p + i * sc] = fmaf(A[4 * i], r0, fmaf(A[4 * i + 1], r1, fmaf(A[4 * i + 2], r2, A[4 * i + 3])));
}

// One step of a recursive-halving warp reduction: lanes with bit `OFF` set keep the upper half of v, the others the lower half,
// and each adds its partner's copy of the half it keeps.  After the five steps of 96 -> 3, lane l holds the warp sums of
// entries 3l .. 3l + 2.
template <int N, int OFF>
__device__ __forceinline__ void halve(float* v, int lane) {
    const bool up = lane & OFF;
#pragma unroll
    for (int k = 0; k < N / 2; ++k) {
        const float send = up ? v[k] : v[k + N / 2];
        const float keep = up ? v[k + N / 2] : v[k];
        v[k] = keep + __shfl_xor_sync(0xffffffffu, send, OFF);
    }
}

__global__ void __launch_bounds__(BT * BT) slice_bwd_kernel(int n_grids, int L, int gh, int gw, const float* __restrict__ grids,
                                                            int height, int width, const float* __restrict__ xy,
                                                            const float* __restrict__ rgb, int64_t sb, int64_t sy, int64_t sx,
                                                            int64_t sc, const int64_t* __restrict__ grid_idx, int n_idx,
                                                            const float* __restrict__ v_out, float* __restrict__ v_rgb,
                                                            float* __restrict__ v_grids) {
    __shared__ float s_acc[BOX_CAP];
    __shared__ int s_box[4];    // x min, x max, y min, y max of the cells touched
    const int tid = threadIdx.y * BT + threadIdx.x, lane = tid & 31;
    const int x = blockIdx.x * BT + threadIdx.x, y = blockIdx.y * BT + threadIdx.y, b = blockIdx.z;
    const bool inside = x < width && y < height;
    const int64_t g = grid_of(grid_idx, n_idx, b);
    const int64_t p = sb * b + sy * y + sx * x;
    if (g < 0 || g >= n_grids) {     // uniform over the CTA
        if (inside && v_rgb) v_rgb[p] = v_rgb[p + sc] = v_rgb[p + 2 * sc] = __int_as_float(0x7fffffff);
        return;
    }
    const int64_t plane = int64_t(L) * gh * gw;
    Sample s;
    float r[3] = {0.f, 0.f, 0.f}, go[3] = {0.f, 0.f, 0.f};
    if (inside) {
#pragma unroll
        for (int i = 0; i < 3; ++i) { r[i] = __ldg(rgb + p + i * sc); go[i] = __ldg(v_out + p + i * sc); }
        const int64_t q = (int64_t(b) * height + y) * width + x;
        s = make_sample(__ldg(xy + 2 * q), __ldg(xy + 2 * q + 1), r[0], r[1], r[2], L, gh, gw);
        if (v_rgb) {
            float A[12], dA[12];
            interpolate(grids + g * 12 * plane, plane, s, gh, gw, A, dA);
            float dgray = 0.f;
#pragma unroll
            for (int i = 0; i < 3; ++i)
                dgray += go[i] * (dA[4 * i] * r[0] + dA[4 * i + 1] * r[1] + dA[4 * i + 2] * r[2] + dA[4 * i + 3]);
            dgray *= s.dgray;
            const float gw3[3] = {GW0, GW1, GW2};
#pragma unroll
            for (int j = 0; j < 3; ++j) v_rgb[p + j * sc] = go[0] * A[j] + go[1] * A[4 + j] + go[2] * A[8 + j] + dgray * gw3[j];
        }
    } else {
        s.x0 = s.y0 = s.z0 = s.dx = s.dy = s.dz = 0;
#pragma unroll
        for (int k = 0; k < 8; ++k) s.w[k] = 0.f;
    }
    if (!v_grids) return;

    if (tid == 0) { s_box[0] = s_box[2] = 0x7fffffff; s_box[1] = s_box[3] = -1; }
    __syncthreads();
    if (inside) {
        atomicMin(&s_box[0], s.x0); atomicMax(&s_box[1], s.x0 + s.dx);
        atomicMin(&s_box[2], s.y0); atomicMax(&s_box[3], s.y0 + s.dy);
    }
    __syncthreads();
    const int bx0 = s_box[0], by0 = s_box[2], bw = s_box[1] - bx0 + 1, bh = s_box[3] - by0 + 1;
    if (bw <= 0) return;                 // no pixel of this CTA lies in the image (uniform)
    const int box = bw * bh * L * 12;
    float* Vg = v_grids + g * 12 * plane;
    const float rr[4] = {r[0], r[1], r[2], 1.f};

    if (box > BOX_CAP) {                 // scattered coordinates: every pixel adds its 96 terms to global memory
        if (!inside) return;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int64_t off = corner_offset(s, k, gh, gw);
#pragma unroll
            for (int c = 0; c < 12; ++c) atomicAdd(Vg + c * plane + off, s.w[k] * go[c >> 2] * rr[c & 3]);
        }
        return;
    }

    for (int e = tid; e < box; e += BT * BT) s_acc[e] = 0.f;
    __syncthreads();
    // lanes that share a lower corner share all eight corners (dx, dy, dz follow from it): sum their 96 terms across the warp,
    // one group of lanes at a time, then three shared-memory adds per lane
    const int key = inside ? (s.z0 * gh + s.y0) * gw + s.x0 : -1;
    unsigned pending = __ballot_sync(0xffffffffu, inside);
    while (pending) {
        const int leader = __ffs(pending) - 1;
        const int lkey = __shfl_sync(0xffffffffu, key, leader);
        const bool member = inside && key == lkey;
        pending &= ~__ballot_sync(0xffffffffu, member);
        float v[96];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const float wk = member ? s.w[k] : 0.f;
#pragma unroll
            for (int c = 0; c < 12; ++c) v[12 * k + c] = wk * go[c >> 2] * rr[c & 3];
        }
        halve<96, 16>(v, lane);
        halve<48, 8>(v, lane);
        halve<24, 4>(v, lane);
        halve<12, 2>(v, lane);
        halve<6, 1>(v, lane);
        const int x0 = __shfl_sync(0xffffffffu, s.x0, leader), y0 = __shfl_sync(0xffffffffu, s.y0, leader);
        const int z0 = __shfl_sync(0xffffffffu, s.z0, leader);
        const int dx = __shfl_sync(0xffffffffu, s.dx, leader), dy = __shfl_sync(0xffffffffu, s.dy, leader);
        const int dz = __shfl_sync(0xffffffffu, s.dz, leader);
        const int k = lane >> 2;         // entries 3 lane .. 3 lane + 2 = corner lane / 4, channels 3 (lane % 4) + t
        const int cx = x0 + (k & 1) * dx - bx0, cy = y0 + ((k >> 1) & 1) * dy - by0, cz = z0 + ((k >> 2) & 1) * dz;
#pragma unroll
        for (int t = 0; t < 3; ++t) {
            const int c = 3 * (lane & 3) + t;
            atomicAdd(&s_acc[((c * L + cz) * bh + cy) * bw + cx], v[t]);
        }
    }
    __syncthreads();
    for (int e = tid; e < box; e += BT * BT) {
        const int cx = e % bw, cy = (e / bw) % bh, cz = (e / (bw * bh)) % L, c = e / (bw * bh * L);
        atomicAdd(Vg + c * plane + (int64_t(cz) * gh + by0 + cy) * gw + bx0 + cx, s_acc[e]);
    }
}

struct TvWeights { float z, y, x; };    // 1 / (n * max(numel per grid of the diff slice, 1)) per axis

__global__ void __launch_bounds__(TV_THREADS) tv_fwd_kernel(int64_t total, int L, int gh, int gw, TvWeights w,
                                                            const float* __restrict__ grids, float* __restrict__ partials) {
    __shared__ float s_red[TV_THREADS / 32];
    const int64_t e = int64_t(blockIdx.x) * TV_THREADS + threadIdx.x;
    float acc = 0.f;
    if (e < total) {
        const int ix = int(e % gw);
        const int64_t t = e / gw;
        const int iy = int(t % gh), iz = int((t / gh) % L);
        const float v = __ldg(grids + e);
        float d;
        if (ix + 1 < gw) { d = __ldg(grids + e + 1) - v; acc = fmaf(w.x * d, d, acc); }
        if (iy + 1 < gh) { d = __ldg(grids + e + gw) - v; acc = fmaf(w.y * d, d, acc); }
        if (iz + 1 < L) { d = __ldg(grids + e + int64_t(gh) * gw) - v; acc = fmaf(w.z * d, d, acc); }
    }
    acc = warp_sum(acc);
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
#pragma unroll
        for (int i = 0; i < TV_THREADS / 32; ++i) t += s_red[i];
        partials[blockIdx.x] = t;
    }
}

// v = up * d tv / d x: each squared difference (b - a)^2 w gives 2 w (a - b) to a and 2 w (b - a) to b
__global__ void __launch_bounds__(TV_THREADS) tv_bwd_kernel(int64_t total, int L, int gh, int gw, TvWeights w,
                                                            const float* __restrict__ grids, const float* __restrict__ v_tv,
                                                            float* __restrict__ v_grids) {
    const int64_t e = int64_t(blockIdx.x) * TV_THREADS + threadIdx.x;
    if (e >= total) return;
    const int ix = int(e % gw);
    const int64_t t = e / gw;
    const int iy = int(t % gh), iz = int((t / gh) % L);
    const int64_t sz = int64_t(gh) * gw;
    const float v = __ldg(grids + e);
    float acc = 0.f;
    if (ix > 0) acc = fmaf(w.x, v - __ldg(grids + e - 1), acc);
    if (ix + 1 < gw) acc = fmaf(w.x, v - __ldg(grids + e + 1), acc);
    if (iy > 0) acc = fmaf(w.y, v - __ldg(grids + e - gw), acc);
    if (iy + 1 < gh) acc = fmaf(w.y, v - __ldg(grids + e + gw), acc);
    if (iz > 0) acc = fmaf(w.z, v - __ldg(grids + e - sz), acc);
    if (iz + 1 < L) acc = fmaf(w.z, v - __ldg(grids + e + sz), acc);
    v_grids[e] = 2.f * __ldg(v_tv) * acc;
}

TvWeights tv_weights(int n, int channels, int L, int gh, int gw) {
    const double per_grid = double(channels) * L * gh * gw;
    auto w = [&](int size) { return float(1.0 / (double(n) * fmax(per_grid / size * (size - 1), 1.0))); };
    return {w(L), w(gh), w(gw)};
}

}  // namespace

int launch_bilagrid_slice_fwd(int n_grids, int L, int gh, int gw, const float* grids, int batch, int height, int width, const float* xy,
                              const float* rgb, int64_t sb, int64_t sy, int64_t sx, int64_t sc, const int64_t* grid_idx, int n_idx,
                              float* out, cudaStream_t s) {
    if (int64_t(batch) * height * width == 0) return B200GS_OK;
    slice_fwd_kernel<<<dim3(div_up(width, BT), div_up(height, BT), batch), dim3(BT, BT), 0, s>>>(
        n_grids, L, gh, gw, grids, height, width, xy, rgb, sb, sy, sx, sc, grid_idx, n_idx, out);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

int launch_bilagrid_slice_bwd(int n_grids, int L, int gh, int gw, const float* grids, int batch, int height, int width, const float* xy,
                              const float* rgb, int64_t sb, int64_t sy, int64_t sx, int64_t sc, const int64_t* grid_idx, int n_idx,
                              const float* v_out, float* v_rgb, float* v_grids, cudaStream_t s) {
    if (int64_t(batch) * height * width == 0 || (!v_rgb && !v_grids)) return B200GS_OK;
    slice_bwd_kernel<<<dim3(div_up(width, BT), div_up(height, BT), batch), dim3(BT, BT), 0, s>>>(
        n_grids, L, gh, gw, grids, height, width, xy, rgb, sb, sy, sx, sc, grid_idx, n_idx, v_out, v_rgb, v_grids);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

int64_t bilagrid_tv_blocks(int n, int channels, int L, int gh, int gw) {
    return div_up64(int64_t(n) * channels * L * gh * gw, TV_THREADS);
}

int launch_bilagrid_tv_fwd(int n, int channels, int L, int gh, int gw, const float* grids, float* partials, cudaStream_t s) {
    const int64_t total = int64_t(n) * channels * L * gh * gw;
    if (total == 0) return B200GS_OK;
    tv_fwd_kernel<<<(unsigned)div_up64(total, TV_THREADS), TV_THREADS, 0, s>>>(total, L, gh, gw, tv_weights(n, channels, L, gh, gw),
                                                                                grids, partials);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

int launch_bilagrid_tv_bwd(int n, int channels, int L, int gh, int gw, const float* grids, const float* v_tv, float* v_grids,
                           cudaStream_t s) {
    const int64_t total = int64_t(n) * channels * L * gh * gw;
    if (total == 0) return B200GS_OK;
    tv_bwd_kernel<<<(unsigned)div_up64(total, TV_THREADS), TV_THREADS, 0, s>>>(total, L, gh, gw, tv_weights(n, channels, L, gh, gw),
                                                                                grids, v_tv, v_grids);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

}  // namespace b200gs
