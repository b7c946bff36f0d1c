// Transient visibility map of the reference's in-the-wild renderer (internal/renderers/gsplat_appearance_embedding_visibility_map_
// renderer.py: Model.visibility_forward :140-157) and its masked loss (internal/metrics/visibility_map_metrics.py).
//   * K32 uv_grid_fwd_kernel: tiny-cuda-nn's 2-D DenseGrid encoding (linear interpolation, 2 features per level) of every pixel's
//     (u, v) = (x / (W - 1), y / (H - 1)), or of given coordinates; the image's grid is the one the appearance id, read on the
//     device, selects from a device table of grid pointers.  Per level l, with the host's fp32 scale_l = exp2f(l log2f(s)) base - 1:
//         res_l = ceil(scale_l) + 1, size_l = next_multiple(res_l^2, 8), pos = fmaf(scale_l, u, 0.5f), cell = floor(pos),
//         frac = pos - cell; the 4 corners in bit order (bit 0: x), weight = (frac or 1 - frac in x) * (.. in y),
//         vertex = (cx + cy res_l) % size_l, enc[2 l + f] = sum of weight * grid[2 (offset_l + vertex) + f].
//     The last pixel column and row reach corner res_l whenever scale_l has a fractional part >= 0.5 (or none); the % wraps it.
//   * K33 uv_grid_bwd_kernel: v_grid of the pixel grid without atomics: one warp per vertex gathers, over the (at most four) corner
//     coordinates the % maps to it, the box of pixels whose cells have that corner, with K32's float formula for every weight, in a
//     fixed order.  uv_grid_scatter_kernel is the backward of given coordinates (float atomics: not bit-reproducible).
//   * K34 vis_loss_fwd_kernel / K35 vis_loss_bwd_kernel: L1 + SSIM (ssim.cuh, the reference ssim.py window K9/K10 use) of a' = w a and b' = w b,
//     w = visibility * mask, plus f mean((1 - visibility)^2).  K34 writes the derivative maps d ssim / d mu_a, d E[a^2] (= d E[b^2]),
//     d E[ab] and, when the visibility needs a gradient, d mu_b, and per-CTA partials of |a' - b'|, SSIM and (1 - v)^2.  K35 (one CTA
//     per tile, the three channels in turn) writes v_image = w dL/da' and v_visibility = mask sum_c (dL/da' a + dL/db' b)
//     - 2 f (1 - v) / (H W).
#include <algorithm>
#include <cmath>

#include "ssim.cuh"

namespace b200gs {

namespace {

constexpr int UV_MAX_LEVELS = 16;

struct GridLevels {
    int n, total;                                             // levels; vertices of all levels
    float scale[UV_MAX_LEVELS];
    int res[UV_MAX_LEVELS], size[UV_MAX_LEVELS], offset[UV_MAX_LEVELS];   // offset in vertices
};

// The level table of g (n_levels 1..16, base_resolution >= 1, per_level_scale >= 1, checked by the caller), or false when the grid
// cannot be addressed: a scale that is not finite, a grid of more than INT32_MAX floats, or a corner cx + cy res_l (cx, cy <= res_l)
// past K32/K33's uint32 vertex arithmetic.  The sizes are summed in int64_t: in int, res_l^2 and the total wrap for large grids, and
// a wrapped total can pass the cap while the size table no longer describes the allocation.
bool grid_levels(const B200gsUvGrid& g, GridLevels& L) {
    L = GridLevels{};
    L.n = g.n_levels;
    const float lg = std::log2(g.per_level_scale);
    int64_t total = 0;
    for (int l = 0; l < g.n_levels; ++l) {
        const float scale = std::exp2(float(l) * lg) * float(g.base_resolution) - 1.f;
        if (!std::isfinite(scale) || scale >= 32768.f) return false;        // res_l^2 alone would pass the float cap
        const int64_t res = int64_t(std::ceil(scale)) + 1;
        const int64_t size = (res * res + 7) / 8 * 8;
        if (res + res * res > int64_t(UINT32_MAX)) return false;            // implied by the cap below; kept as the kernels' bound
        L.scale[l] = scale;
        L.res[l] = int(res);
        L.size[l] = int(size);
        L.offset[l] = int(total);
        total += size;
        if (2 * total > INT32_MAX) return false;
    }
    L.total = int(total);
    return true;
}

// the pixel's coordinate along one axis, as the reference's fp32 arange / (n - 1)
__device__ __forceinline__ float pixel_coord(int i, int n) { return __fdiv_rn(float(i), float(n - 1)); }

struct Axis {
    uint32_t cell;
    float frac;
};

__device__ __forceinline__ Axis axis(float scale, float u) {
    const float pos = fmaf(scale, u, 0.5f);
    const float c = floorf(pos);
    return {uint32_t(int(c)), pos - c};
}

__global__ void __launch_bounds__(256) uv_grid_fwd_kernel(const GridLevels g, int width, int height, const float* __restrict__ uv, int64_t n,
                                                          const float* const* __restrict__ grids, int n_grids, const int64_t* id_dev,
                                                          int64_t id_host, float* __restrict__ enc) {
    const int64_t row = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (row >= n) return;
    const int64_t id = id_dev ? __ldg(id_dev) : id_host;
    float2* out = reinterpret_cast<float2*>(enc + row * 2 * g.n);
    if (id < 0 || id >= n_grids) {
        for (int l = 0; l < g.n; ++l) out[l] = make_float2(__int_as_float(0x7fc00000), __int_as_float(0x7fc00000));
        return;
    }
    const float2* P = reinterpret_cast<const float2*>(grids[id]);
    float u, v;
    if (uv) {
        u = __ldg(uv + 2 * row);
        v = __ldg(uv + 2 * row + 1);
    } else {
        const int y = int(row / width), x = int(row - int64_t(y) * width);
        u = pixel_coord(x, width);
        v = pixel_coord(y, height);
    }
    for (int l = 0; l < g.n; ++l) {
        const Axis ax = axis(g.scale[l], u), ay = axis(g.scale[l], v);
        const uint32_t res = g.res[l], size = g.size[l];
        float2 acc = make_float2(0.f, 0.f);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float w = ((k & 1) ? ax.frac : 1.f - ax.frac) * ((k & 2) ? ay.frac : 1.f - ay.frac);
            const uint32_t vert = ((ax.cell + (k & 1)) + (ay.cell + (k >> 1)) * res) % size;
            const float2 p = __ldg(P + g.offset[l] + vert);
            acc.x = fmaf(w, p.x, acc.x);
            acc.y = fmaf(w, p.y, acc.y);
        }
        out[l] = acc;
    }
}

// [lo, hi]: the pixels along an axis of n pixels whose cell is c - 1 or c (the cells that have corner c); empty when lo > hi
__device__ __forceinline__ void corner_range(float scale, int n, uint32_t c, int& lo, int& hi) {
    // the cell is non-decreasing in the pixel index: first pixel with cell >= c - 1, last with cell <= c
    int a = 0, b = n;
    while (a < b) {
        const int m = (a + b) >> 1;
        if (int(axis(scale, pixel_coord(m, n)).cell) >= int(c) - 1) b = m; else a = m + 1;
    }
    lo = a;
    a = 0; b = n;
    while (a < b) {
        const int m = (a + b) >> 1;
        if (int(axis(scale, pixel_coord(m, n)).cell) > int(c)) b = m; else a = m + 1;
    }
    hi = a - 1;
}

__global__ void __launch_bounds__(256) uv_grid_bwd_kernel(const GridLevels g, int width, int height, const float* __restrict__ v_enc,
                                                          float* __restrict__ v_grid) {
    const int vid = int(blockIdx.x) * (blockDim.x >> 5) + int(threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (vid >= g.total) return;
    int l = 0;
    while (l + 1 < g.n && vid >= g.offset[l + 1]) ++l;
    const uint32_t vert = vid - g.offset[l], res = g.res[l], size = g.size[l];
    const float scale = g.scale[l];
    const uint32_t cmax = axis(scale, 1.f).cell + 1;          // the largest corner coordinate the pixel grid reaches
    float acc0 = 0.f, acc1 = 0.f;
    // the corner coordinates (cx, cy), cx, cy <= cmax <= res, with (cx + cy res) % size == vert: cx + cy res is vert or
    // vert + size (< 2 size), written as (j % res, j / res) or, when j % res == 0, as (res, j / res - 1)
    for (int q = 0; q < 4; ++q) {
        const uint32_t j = vert + (q >> 1) * size;
        uint32_t cx = j % res, cy = j / res;
        if (q & 1) {
            if (cx != 0 || cy == 0) continue;
            cx = res; cy -= 1;
        }
        if (cx > cmax || cy > cmax) continue;
        int x0, x1, y0, y1;
        corner_range(scale, width, cx, x0, x1);
        corner_range(scale, height, cy, y0, y1);
        if (x0 > x1 || y0 > y1) continue;
        const int bw = x1 - x0 + 1;
        const int64_t count = int64_t(bw) * (y1 - y0 + 1);
        for (int64_t k = lane; k < count; k += 32) {
            const int y = y0 + int(k / bw), x = x0 + int(k - int64_t(k / bw) * bw);
            const Axis ax = axis(scale, pixel_coord(x, width)), ay = axis(scale, pixel_coord(y, height));
            const bool bx = ax.cell != cx, by = ay.cell != cy;          // this corner is the cell's +1 corner along the axis
            const float w = (bx ? ax.frac : 1.f - ax.frac) * (by ? ay.frac : 1.f - ay.frac);
            const float2 d = __ldg(reinterpret_cast<const float2*>(v_enc + (int64_t(y) * width + x) * 2 * g.n) + l);
            acc0 = fmaf(w, d.x, acc0);
            acc1 = fmaf(w, d.y, acc1);
        }
    }
    acc0 = warp_sum(acc0);
    acc1 = warp_sum(acc1);
    if (lane == 0) reinterpret_cast<float2*>(v_grid)[vid] = make_float2(acc0, acc1);
}

__global__ void __launch_bounds__(256) uv_grid_scatter_kernel(const GridLevels g, const float* __restrict__ uv, int64_t n,
                                                              const float* __restrict__ v_enc, float* __restrict__ v_grid) {
    const int64_t row = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (row >= n) return;
    const float u = __ldg(uv + 2 * row), v = __ldg(uv + 2 * row + 1);
    for (int l = 0; l < g.n; ++l) {
        const Axis ax = axis(g.scale[l], u), ay = axis(g.scale[l], v);
        const uint32_t res = g.res[l], size = g.size[l];
        const float2 d = __ldg(reinterpret_cast<const float2*>(v_enc + row * 2 * g.n) + l);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float w = ((k & 1) ? ax.frac : 1.f - ax.frac) * ((k & 2) ? ay.frac : 1.f - ay.frac);
            const uint32_t vert = ((ax.cell + (k & 1)) + (ay.cell + (k >> 1)) * res) % size;
            atomicAdd(v_grid + 2 * (g.offset[l] + vert), w * d.x);
            atomicAdd(v_grid + 2 * (g.offset[l] + vert) + 1, w * d.y);
        }
    }
}

// ---- K34 / K35 ----------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float weight_at(const float* vis, const uint8_t* mask, int64_t p) {
    const float v = __ldg(vis + p);
    return mask && __ldg(mask + p) == 0 ? 0.f : v;       // w = visibility * mask (mask uint8: 0 or 1)
}

__global__ void __launch_bounds__(LT * LT) vis_loss_fwd_kernel(int width, int height, const float* __restrict__ img,
                                                               const float* __restrict__ gt, const float* __restrict__ vis,
                                                               const uint8_t* __restrict__ mask, int vis_grad, float* __restrict__ dmaps,
                                                               float* __restrict__ partials) {
    __shared__ float s_a[LE][LE], s_b[LE][LE];
    __shared__ float s_h[5][LE][LT];
    __shared__ float s_red[LT * LT / 32][3];
    const int c = blockIdx.z;
    const int x0 = blockIdx.x * LT, y0 = blockIdx.y * LT;
    const int64_t plane = int64_t(width) * height;
    const float* img_c = img + c * plane;
    const float* gt_c = gt + c * plane;
    load_halo(width, height, x0, y0, {s_a}, [=](int, int64_t p) { return __ldg(img_c + p) * weight_at(vis, mask, p); });
    load_halo(width, height, x0, y0, {s_b}, [=](int, int64_t p) { return __ldg(gt_c + p) * weight_at(vis, mask, p); });
    __syncthreads();
    blur_moments_h(c_ssim_win, s_a, s_b, s_h);
    __syncthreads();
    const int lx = threadIdx.x % LT, ly = threadIdx.x / LT;
    const int x = x0 + lx, y = y0 + ly;
    float m[5];
    blur_moments_v(c_ssim_win, s_h, ly, lx, m);
    float acc[3] = {0.f, 0.f, 0.f};         // |a' - b'|, SSIM, (1 - v)^2
    if (x < width && y < height) {
        const float a = s_a[ly + HALO][lx + HALO], b = s_b[ly + HALO][lx + HALO];
        const SsimTerms t = ssim_terms<0>(m, SSIM_C1, SSIM_C2);
        acc[0] = fabsf(a - b);
        acc[1] = t.ssim;
        const int64_t pix = int64_t(y) * width + x;
        if (c == 0) {
            const float r = 1.f - __ldg(vis + pix);
            acc[2] = r * r;
        }
        const int64_t p = c * plane + pix, stride = 3 * plane;
        dmaps[p] = t.d_mu;
        dmaps[stride + p] = t.d_xx;
        dmaps[2 * stride + p] = t.d_ab;
        if (vis_grad) dmaps[3 * stride + p] = ssim_terms<1>(m, SSIM_C1, SSIM_C2).d_mu;
    }
    cta_sum_row(acc, s_red, threadIdx.x,
                [&] { return partials + 3 * ((int64_t(blockIdx.z) * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x); });
}

__global__ void __launch_bounds__(LT * LT) vis_loss_bwd_kernel(int width, int height, const float* __restrict__ img,
                                                               const float* __restrict__ gt, const float* __restrict__ vis,
                                                               const uint8_t* __restrict__ mask, const float* __restrict__ dmaps,
                                                               float lambda, float reg, const float* __restrict__ v_loss,
                                                               float* __restrict__ v_img, float* __restrict__ v_vis) {
    __shared__ float s_m[3][LE][LE];
    __shared__ float s_h[3][LE][LT];
    const int x0 = blockIdx.x * LT, y0 = blockIdx.y * LT;
    const int64_t plane = int64_t(width) * height, stride = 3 * plane;
    const int lx = threadIdx.x % LT, ly = threadIdx.x / LT;
    const int x = x0 + lx, y = y0 + ly;
    const bool inside = x < width && y < height;
    const int64_t pix = int64_t(y) * width + x;
    const float inv_n = 1.f / (3.f * float(width) * float(height));
    const float up = v_loss ? __ldg(v_loss) : 1.f;
    const float w = inside ? weight_at(vis, mask, pix) : 0.f;
    float dv = 0.f;
    for (int c = 0; c < 3; ++c) {
        float g[3], gb = 0.f;
#pragma unroll
        for (int m = 0; m < 3; ++m) {
            const float* map = dmaps + m * stride + c * plane;
            load_halo(width, height, x0, y0, {s_m[m]}, [=](int, int64_t p) { return __ldg(map + p); });
        }
        __syncthreads();
        blur_maps_h(c_ssim_win, s_m, s_h);
        __syncthreads();
        blur_maps_v(c_ssim_win, s_h, ly, lx, g);
        if (v_vis) {           // d ssim / d mu_b: the one map the b' operand adds (d E[b^2] is the d E[a^2] map)
            __syncthreads();
            const float* map = dmaps + 3 * stride + c * plane;
            load_halo(width, height, x0, y0, {s_m[0]}, [=](int, int64_t p) { return __ldg(map + p); });
            __syncthreads();
            for (int i = threadIdx.x; i < LE * LT; i += LT * LT) {
                const int r = i / LT, q = i - r * LT;
                float h = 0.f;
#pragma unroll
                for (int k = 0; k < TAPS; ++k) h = fmaf(c_ssim_win[k], s_m[0][r][q + k], h);
                s_h[0][r][q] = h;
            }
            __syncthreads();
#pragma unroll
            for (int k = 0; k < TAPS; ++k) gb = fmaf(c_ssim_win[k], s_h[0][ly + k][lx], gb);
        }
        if (inside) {
            const int64_t p = c * plane + pix;
            const float a = __ldg(img + p), b = __ldg(gt + p);
            const float ap = a * w, bp = b * w;
            const float d = ap - bp;
            const float sgn = d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f);          // torch.abs' subgradient at 0 is 0
            const float da = up * inv_n * ((1.f - lambda) * sgn - lambda * ssim_grad(g, ap, bp));
            v_img[p] = w * da;
            if (v_vis) {
                const float db = up * inv_n * (-(1.f - lambda) * sgn - lambda * (gb + 2.f * bp * g[1] + ap * g[2]));
                dv += da * a + db * b;
            }
        }
        __syncthreads();       // s_m and s_h are reloaded for the next channel
    }
    if (v_vis && inside) {
        const float keep = mask && __ldg(mask + pix) == 0 ? 0.f : 1.f;
        v_vis[pix] = keep * dv - up * 2.f * reg * (1.f - __ldg(vis + pix)) / (float(width) * float(height));
    }
}

// the level table of a supported grid into L; false for any other
bool uv_grid_ok(const B200gsUvGrid* g, GridLevels& L) {
    return g && g->n_levels >= 1 && g->n_levels <= UV_MAX_LEVELS && g->base_resolution >= 1 && g->per_level_scale >= 1.f &&
           std::isfinite(g->per_level_scale) && grid_levels(*g, L);
}

// shared by the forward and the backward; returns the error code, or 0 when the arguments are valid and L holds the level table
int check_uv_grid(const char* fn, const B200gsUvGrid* grid, int32_t width, int32_t height, const float* uv, int64_t n, GridLevels& L) {
    if (!uv_grid_ok(grid, L))
        return fail(fn, "bad grid: n_levels 1..16, base_resolution >= 1, per_level_scale >= 1, at most INT32_MAX floats");
    if (uv == nullptr) {
        if (width < 2 || height < 2) return fail(fn, "the pixel grid needs width and height >= 2 (u = x / (width - 1))");
        if (int64_t(width) * height > INT32_MAX) return fail(fn, "image too large");
    } else if (n < 0 || n > INT32_MAX) {
        return fail(fn, "n out of range");
    }
    return 0;
}

// the grid is (ceil(W/LT), ceil(H/LT), 3): ceil(H/LT) is at most 65535
bool vis_loss_size_ok(int32_t width, int32_t height) {
    return width >= 1 && height >= 1 && height <= 65535 * LT && int64_t(width) * height <= INT32_MAX / 4;
}

int64_t vis_loss_blocks(int width, int height) { return 3 * int64_t(div_up(width, LT)) * div_up(height, LT); }

// the workspace holds the derivative maps, then the per-CTA partials
size_t vis_loss_workspace_bytes(int width, int height, bool vis_grad) {
    return (size_t(vis_grad ? 4 : 3) * 3 * size_t(width) * height + 3 * size_t(vis_loss_blocks(width, height))) * sizeof(float);
}

// shared by the forward and the backward; returns the error code, or 0 when the arguments are valid
int check_vis_loss(const char* fn, int32_t width, int32_t height, const float* image, const float* gt, const float* visibility,
                   const void* workspace, size_t workspace_bytes, bool vis_grad) {
    if (width < 1 || height < 1) return fail(fn, "image size must be >= 1");
    if (!vis_loss_size_ok(width, height)) return fail(fn, "image too large");
    if (!(image && gt && visibility && workspace)) return fail(fn, "NULL pointer");
    if (workspace_bytes < vis_loss_workspace_bytes(width, height, vis_grad)) return workspace_too_small(fn);
    return 0;
}

}  // namespace

}  // namespace b200gs

using namespace b200gs;

extern "C" {

int64_t b200gs_uv_grid_params(const B200gsUvGrid* grid) {
    GridLevels g;
    return uv_grid_ok(grid, g) ? 2 * int64_t(g.total) : 0;
}

int b200gs_uv_grid_fwd(const B200gsUvGrid* grid, int32_t width, int32_t height, const float* uv, int64_t n, const float* const* grids,
                       int32_t n_grids, const int64_t* appearance_id, int64_t host_appearance_id, float* enc, void* stream) {
    GridLevels g;
    if (int rc = check_uv_grid(__func__, grid, width, height, uv, n, g)) return rc;
    B200GS_CHECK_ARG(n_grids >= 1, "n_grids must be >= 1");
    B200GS_CHECK_ARG(grids && enc, "NULL pointer");
    B200GS_CHECK_ARG((reinterpret_cast<uintptr_t>(enc) & 7u) == 0, "enc must be 8-byte aligned");
    if (!uv) n = int64_t(width) * height;
    if (n == 0) return B200GS_OK;
    uv_grid_fwd_kernel<<<unsigned(div_up64(n, 256)), 256, 0, (cudaStream_t)stream>>>(g, width, height, uv, n, grids, n_grids, appearance_id,
                                                                                     host_appearance_id, enc);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

int b200gs_uv_grid_bwd(const B200gsUvGrid* grid, int32_t width, int32_t height, const float* uv, int64_t n, const float* v_enc,
                       float* v_grid, void* stream) {
    GridLevels g;
    if (int rc = check_uv_grid(__func__, grid, width, height, uv, n, g)) return rc;
    B200GS_CHECK_ARG(v_enc && v_grid, "NULL pointer");
    B200GS_CHECK_ARG(((reinterpret_cast<uintptr_t>(v_enc) | reinterpret_cast<uintptr_t>(v_grid)) & 7u) == 0,
                     "v_enc and v_params must be 8-byte aligned");
    const cudaStream_t s = (cudaStream_t)stream;
    if (uv) {
        B200GS_CUDA(cudaMemsetAsync(v_grid, 0, size_t(g.total) * 2 * sizeof(float), s));
        if (n == 0) return B200GS_OK;
        uv_grid_scatter_kernel<<<unsigned(div_up64(n, 256)), 256, 0, s>>>(g, uv, n, v_enc, v_grid);
    } else {
        uv_grid_bwd_kernel<<<div_up(g.total, 8), 256, 0, s>>>(g, width, height, v_enc, v_grid);
    }
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

int64_t b200gs_vis_loss_blocks(int32_t width, int32_t height) { return vis_loss_size_ok(width, height) ? vis_loss_blocks(width, height) : 0; }

size_t b200gs_vis_loss_workspace_bytes(int32_t width, int32_t height, int32_t vis_grad) {
    return vis_loss_size_ok(width, height) ? vis_loss_workspace_bytes(width, height, vis_grad != 0) : 0;
}

int b200gs_vis_loss_fwd(int32_t width, int32_t height, const float* image, const float* gt, const float* visibility, const uint8_t* mask,
                        int32_t vis_grad, void* workspace, size_t workspace_bytes, void* stream) {
    if (int rc = check_vis_loss(__func__, width, height, image, gt, visibility, workspace, workspace_bytes, vis_grad != 0)) return rc;
    float* ws = static_cast<float*>(workspace);
    const dim3 grid(div_up(width, LT), div_up(height, LT), 3);
    float* partials = ws + size_t(vis_grad ? 4 : 3) * 3 * size_t(width) * height;
    vis_loss_fwd_kernel<<<grid, LT * LT, 0, (cudaStream_t)stream>>>(width, height, image, gt, visibility, mask, vis_grad != 0, ws, partials);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

int b200gs_vis_loss_bwd(int32_t width, int32_t height, const float* image, const float* gt, const float* visibility, const uint8_t* mask,
                        const void* workspace, size_t workspace_bytes, float lambda_dssim, float vis_reg_factor, const float* v_loss,
                        float* v_image, float* v_visibility, void* stream) {
    if (int rc = check_vis_loss(__func__, width, height, image, gt, visibility, workspace, workspace_bytes, v_visibility != nullptr))
        return rc;
    B200GS_CHECK_ARG(v_image, "NULL v_image");
    const dim3 grid(div_up(width, LT), div_up(height, LT));
    vis_loss_bwd_kernel<<<grid, LT * LT, 0, (cudaStream_t)stream>>>(width, height, image, gt, visibility, mask,
                                                                    static_cast<const float*>(workspace), lambda_dssim, vis_reg_factor,
                                                                    v_loss, v_image, v_visibility);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

}  // extern "C"
