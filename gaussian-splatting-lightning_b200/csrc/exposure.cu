// Learned exposure correction, the per-image colour transform of internal/output_processors/exposure.py (ExposureProcessorModule,
// :112-143) that runs between the render and the loss on every training step.  For one view, with a = sigmoid(P[id]) (P is
// [n_appearances, 4 | 7]) and the shade map S[0] (s x s):
//     M      = sigmoid(S[0]) / clamp_min(max(sigmoid(S[0])), 1e-4)            (the max is detached)
//     m(y,x) = bilinear, align_corners=True, of M at (y (s-1)/(H-1), x (s-1)/(W-1))      (torch's upsample_bilinear2d)
//     x_c    = (a_c max_gray) (r_c m) [+ 2 a_{3+c} - 1]
//     c      = clamp(x, 0, 1), straight through (the gradient passes as identity)
//     out    = (c + 1e-5) ^ (a_last max_gamma)
// The reference writes the clamp as x - (x - clamp(x)).detach(), which is clamp(x) exactly for |x| < 2^24.
//   * prep: one CTA; reads the appearance id on the device, writes a, the selected row and (with shade correction) the max and
//     M into the workspace head, so the pixel kernels read M from L2 instead of each CTA re-reducing the map.
//   * fwd: one thread per pixel; render / out through element strides, so the permuted [H,W,3] render is read in place.
//   * bwd: v_render per pixel; the parameter sums as per-CTA partials (fixed-order warp and CTA reductions); v_m, the gradient of
//     m, per pixel into the workspace.
//   * reduce: CTA 0 adds the partials in block order and writes the whole v_P (rows other than id exactly zero); the other CTAs
//     gather v_S one warp per cell over the pixel box that references it, in a fixed order: no float atomics anywhere, so two
//     backwards give bit-identical gradients.
// An id outside [0, n_appearances) reads no row: out and v_render are NaN, v_P and v_S zero.
#include "common.cuh"

namespace b200gs {

namespace {

constexpr int BX = 32, BY = 8;          // pixel tile of the fwd / bwd kernels
constexpr int PREP_THREADS = 1024;
constexpr int RED_THREADS = 256;        // reduce: 8 warps, one cell each
constexpr int HEAD = 16;                // workspace floats before M: a[0..6], row (int bits, -1 if invalid), max
constexpr int PARTIAL = 8;              // floats per CTA partial: v_a[0..6] (gamma last), pad

struct ExpoArgs {
    int height, width;
    int64_t sc, sy, sx;
    int n_params, s;                    // s = 0: no shade correction
    float max_gray, max_gamma;
    float ry, rx;                       // torch's align_corners source scales (s - 1) / (H - 1), 0 for a size-1 output
};

__device__ __forceinline__ float sigmoidf(float v) { return 1.f / (1.f + __expf(-v)); }

// torch's upsample_bilinear2d(align_corners=True) source index of one axis: lower cell i0, step d (0 on the last cell), weight l
// of the upper cell
__device__ __forceinline__ void src_axis(float r, int dst, int s, int& i0, int& d, float& l) {
    const float f = r * float(dst);
    i0 = int(f);
    d = i0 < s - 1 ? 1 : 0;
    l = f - float(i0);
}

__device__ __forceinline__ float shade_at(const float* __restrict__ M, const ExpoArgs& g, int y, int x) {
    int y0, dy, x0, dx;
    float ly, lx;
    src_axis(g.ry, y, g.s, y0, dy, ly);
    src_axis(g.rx, x, g.s, x0, dx, lx);
    const float* r0 = M + y0 * g.s + x0;
    const float* r1 = r0 + dy * g.s;
    return (1.f - ly) * ((1.f - lx) * __ldg(r0) + lx * __ldg(r0 + dx)) + ly * ((1.f - lx) * __ldg(r1) + lx * __ldg(r1 + dx));
}

__global__ void __launch_bounds__(PREP_THREADS) exposure_prep_kernel(int n_app, int n_params, const float* __restrict__ P,
                                                                     const int64_t* __restrict__ id_dev, int64_t id_host, int s,
                                                                     const float* __restrict__ S, float* __restrict__ ws) {
    __shared__ float s_max[PREP_THREADS / 32];
    const int t = threadIdx.x;
    const int64_t id = id_dev ? __ldg(id_dev) : id_host;
    const bool valid = id >= 0 && id < n_app;
    if (t < 7) ws[t] = (valid && t < n_params) ? sigmoidf(__ldg(P + id * n_params + t)) : 0.f;
    if (t == 7) ws[7] = __int_as_float(valid ? int(id) : -1);
    if (s == 0) return;
    const int n = s * s;
    float mx = 0.f;                     // sigmoid > 0
    for (int i = t; i < n; i += PREP_THREADS) mx = fmaxf(mx, sigmoidf(__ldg(S + i)));
    mx = warp_reduce<Max>(mx);
    if ((t & 31) == 0) s_max[t >> 5] = mx;
    __syncthreads();
    mx = 0.f;
#pragma unroll
    for (int w = 0; w < PREP_THREADS / 32; ++w) mx = fmaxf(mx, s_max[w]);
    mx = fmaxf(mx, 1e-4f);
    if (t == 0) ws[8] = mx;
    for (int i = t; i < n; i += PREP_THREADS) ws[HEAD + i] = sigmoidf(__ldg(S + i)) / mx;
}

template <bool SHADE>
__global__ void __launch_bounds__(BX * BY) exposure_fwd_kernel(ExpoArgs g, const float* __restrict__ render, const float* __restrict__ ws,
                                                               float* __restrict__ out) {
    const int x = blockIdx.x * BX + threadIdx.x, y = blockIdx.y * BY + threadIdx.y;
    if (x >= g.width || y >= g.height) return;
    const int64_t p = g.sy * y + g.sx * x;
    if (__float_as_int(__ldg(ws + 7)) < 0) {
        out[p] = out[p + g.sc] = out[p + 2 * g.sc] = __int_as_float(0x7fffffff);
        return;
    }
    const float m = SHADE ? shade_at(ws + HEAD, g, y, x) : 1.f;
    const float gamma = __ldg(ws + g.n_params - 1) * g.max_gamma;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        float v = (__ldg(ws + c) * g.max_gray) * (__ldg(render + p + c * g.sc) * m);
        if (g.n_params == 7) v += __ldg(ws + 3 + c) * 2.f - 1.f;
        out[p + c * g.sc] = __powf(fminf(fmaxf(v, 0.f), 1.f) + 1e-5f, gamma);
    }
}

template <bool SHADE>
__global__ void __launch_bounds__(BX * BY) exposure_bwd_kernel(ExpoArgs g, const float* __restrict__ render, const float* __restrict__ v_out,
                                                               const float* __restrict__ ws, float* __restrict__ v_render,
                                                               float* __restrict__ partials, float* __restrict__ v_m) {
    __shared__ float s_red[BX * BY / 32][7];
    const int x = blockIdx.x * BX + threadIdx.x, y = blockIdx.y * BY + threadIdx.y;
    const int tid = threadIdx.y * BX + threadIdx.x;
    const bool valid = __float_as_int(__ldg(ws + 7)) >= 0;
    float acc[7] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};       // d/d a_c, d/d a_{3+c}, d/d gamma
    if (x < g.width && y < g.height) {
        const int64_t p = g.sy * y + g.sx * x;
        if (!valid) {
            v_render[p] = v_render[p + g.sc] = v_render[p + 2 * g.sc] = __int_as_float(0x7fffffff);
            if (SHADE) v_m[int64_t(y) * g.width + x] = 0.f;
        } else {
            const float m = SHADE ? shade_at(ws + HEAD, g, y, x) : 1.f;
            const float gamma = __ldg(ws + g.n_params - 1) * g.max_gamma;
            float vm = 0.f;
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float r = __ldg(render + p + c * g.sc), go = __ldg(v_out + p + c * g.sc);
                const float k = __ldg(ws + c) * g.max_gray, t = r * m;
                float v = k * t;
                if (g.n_params == 7) v += __ldg(ws + 3 + c) * 2.f - 1.f;
                const float base = fminf(fmaxf(v, 0.f), 1.f) + 1e-5f;
                const float vx = go * gamma * __powf(base, gamma - 1.f);       // straight through the clamp
                acc[c] = vx * t;
                acc[3 + c] = 2.f * vx;
                acc[6] += go * __powf(base, gamma) * __logf(base);
                const float vt = vx * k;
                v_render[p + c * g.sc] = vt * m;
                vm = fmaf(vt, r, vm);
            }
            if (SHADE) v_m[int64_t(y) * g.width + x] = vm;
        }
    }
    cta_sum_row(acc, s_red, tid, [&] { return partials + int64_t(blockIdx.y * gridDim.x + blockIdx.x) * PARTIAL; });
}

// pixel range [lo, hi] of one axis whose bilinear footprint may include cell i (widened by one; the caller tests membership)
__device__ __forceinline__ void cell_range(float r, int i, int n, int& lo, int& hi) {
    if (r == 0.f) { lo = 0; hi = n - 1; return; }
    lo = max(0, int(floorf(float(i - 1) / r)) - 1);
    hi = int(fminf(ceilf(float(i + 1) / r) + 1.f, float(n - 1)));
}

// weight of cell i in pixel dst's bilinear interpolation along one axis (both terms when the pixel sits on the last cell)
__device__ __forceinline__ float cell_weight(float r, int dst, int s, int i) {
    int i0, d;
    float l;
    src_axis(r, dst, s, i0, d, l);
    return (i0 == i ? 1.f - l : 0.f) + (i0 + d == i ? l : 0.f);
}

__global__ void __launch_bounds__(RED_THREADS) exposure_reduce_kernel(ExpoArgs g, int n_blocks, int n_app, const float* __restrict__ ws,
                                                                      const float* __restrict__ partials, const float* __restrict__ v_m,
                                                                      const float* __restrict__ S, float* __restrict__ v_P,
                                                                      float* __restrict__ v_S) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (blockIdx.x == 0) {              // parameters: warp k adds partial k over the CTAs, each lane a fixed stride, then the warp
        __shared__ float s_v[8];
        if (warp < 7) {
            float t = 0.f;
            for (int b = lane; b < n_blocks; b += 32) t += __ldg(partials + int64_t(b) * PARTIAL + warp);
            t = warp_sum(t);
            if (lane == 0) s_v[warp] = t;
        }
        __syncthreads();
        const int row = __float_as_int(__ldg(ws + 7));
        const int np = g.n_params;
        for (int e = tid; e < n_app * np; e += RED_THREADS) {
            float v = 0.f;
            if (e / np == row) {
                const int k = e % np;
                const float a = __ldg(ws + k);
                const float va = k < 3 ? s_v[k] * g.max_gray : (k == np - 1 ? s_v[6] * g.max_gamma : s_v[k]);
                v = va * (1.f - a) * a;
            }
            v_P[e] = v;
        }
        return;
    }
    const int cell = (blockIdx.x - 1) * (RED_THREADS / 32) + warp;
    if (cell >= g.s * g.s) return;
    const int ci = cell / g.s, cj = cell % g.s;
    int y_lo, y_hi, x_lo, x_hi;
    cell_range(g.ry, ci, g.height, y_lo, y_hi);
    cell_range(g.rx, cj, g.width, x_lo, x_hi);
    float acc = 0.f;
    for (int y = y_lo; y <= y_hi; ++y) {
        const float wy = cell_weight(g.ry, y, g.s, ci);
        if (wy == 0.f) continue;       // uniform over the warp
        const float* row = v_m + int64_t(y) * g.width;
        for (int x = x_lo + lane; x <= x_hi; x += 32) {
            const float wx = cell_weight(g.rx, x, g.s, cj);
            acc = fmaf(wy * wx, __ldg(row + x), acc);
        }
    }
    acc = warp_sum(acc);
    if (lane == 0) {
        const float sg = sigmoidf(__ldg(S + cell));
        v_S[cell] = acc / __ldg(ws + 8) * (1.f - sg) * sg;
    }
}

int64_t pixel_blocks(int height, int width) { return int64_t(div_up(width, BX)) * div_up(height, BY); }

ExpoArgs make_args(int height, int width, int64_t sc, int64_t sy, int64_t sx, int n_params, int s, float max_gray, float max_gamma) {
    ExpoArgs g;
    g.height = height; g.width = width; g.sc = sc; g.sy = sy; g.sx = sx;
    g.n_params = n_params; g.s = s; g.max_gray = max_gray; g.max_gamma = max_gamma;
    // torch's area_pixel_compute_scale in float: (in - 1) / (out - 1), 0 when the output has one pixel
    g.ry = height > 1 ? float(s - 1) / float(height - 1) : 0.f;
    g.rx = width > 1 ? float(s - 1) / float(width - 1) : 0.f;
    return g;
}

// the grid is (ceil(W/BX), ceil(H/BY)): ceil(H/BY) is at most 65535
bool exposure_size_ok(int32_t height, int32_t width, int32_t shade_size) {
    return height >= 1 && width >= 1 && height <= 65535 * BY && int64_t(height) * width <= INT32_MAX && shade_size >= 0 &&
           shade_size <= 4096;
}

size_t exposure_workspace_bytes(int height, int width, int shade_size, bool backward) {
    int64_t floats = HEAD + int64_t(shade_size) * shade_size;
    if (backward) floats += pixel_blocks(height, width) * PARTIAL + (shade_size > 0 ? int64_t(height) * width : 0);
    return size_t(floats) * sizeof(float);
}

// render / out / v_out / v_render [3,H,W] through the element strides (sc, sy, sx); params [n_appearances, n_params] (n_params 4 or
// 7: with bias); the id read from appearance_id when not NULL, else host_appearance_id; shade [s, s] (s = 0: none).  Shared by the
// forward and the backward; returns the error code, or 0 when the arguments are valid
int check_exposure(const char* fn, int32_t channels, int32_t height, int32_t width, const float* render, int64_t sc, int64_t sy, int64_t sx,
                   int32_t n_appearances, int32_t n_params, const float* exposure_params, int32_t shade_size, const float* shade,
                   const void* workspace, size_t workspace_bytes, bool backward, const void* out) {
    if (channels != 3) return fail(fn, "channels must be 3");
    if (height < 1 || width < 1) return fail(fn, "image size must be >= 1");
    if (shade_size < 0) return fail(fn, "negative shade_size");
    if (!exposure_size_ok(height, width, shade_size)) return fail(fn, "image or shade map too large");
    if (sc < 0 || sy < 0 || sx < 0) return fail(fn, "negative stride");
    if (n_appearances < 1) return fail(fn, "n_appearances must be >= 1");
    if (n_params != 4 && n_params != 7) return fail(fn, "n_params must be 4 (no bias) or 7 (with bias)");
    if (!(render && exposure_params && workspace && out) || (shade_size > 0 && !shade)) return fail(fn, "NULL pointer");
    if (workspace_bytes < exposure_workspace_bytes(height, width, shade_size, backward)) return workspace_too_small(fn);
    return 0;
}

}  // namespace

}  // namespace b200gs

using namespace b200gs;

extern "C" {

size_t b200gs_exposure_workspace_bytes(int32_t height, int32_t width, int32_t shade_size, int32_t backward) {
    if (!exposure_size_ok(height, width, shade_size)) return 0;
    return exposure_workspace_bytes(height, width, shade_size, backward != 0);
}

int b200gs_exposure_fwd(int32_t channels, int32_t height, int32_t width, const float* render, int64_t sc, int64_t sy, int64_t sx,
                        int32_t n_appearances, int32_t n_params, const float* exposure_params, const int64_t* appearance_id,
                        int64_t host_appearance_id, int32_t s, const float* shade, float max_gray_scale, float max_gamma,
                        void* workspace, size_t workspace_bytes, float* out, void* stream) {
    if (int rc = check_exposure(__func__, channels, height, width, render, sc, sy, sx, n_appearances, n_params, exposure_params, s, shade,
                                workspace, workspace_bytes, false, out))
        return rc;
    const cudaStream_t st = (cudaStream_t)stream;
    float* ws = static_cast<float*>(workspace);
    const ExpoArgs g = make_args(height, width, sc, sy, sx, n_params, s, max_gray_scale, max_gamma);
    exposure_prep_kernel<<<1, PREP_THREADS, 0, st>>>(n_appearances, n_params, exposure_params, appearance_id, host_appearance_id, s, shade, ws);
    B200GS_LAUNCH_CHECK();
    const dim3 grid(div_up(width, BX), div_up(height, BY)), block(BX, BY);
    if (s > 0) exposure_fwd_kernel<true><<<grid, block, 0, st>>>(g, render, ws, out);
    else exposure_fwd_kernel<false><<<grid, block, 0, st>>>(g, render, ws, out);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

int b200gs_exposure_bwd(int32_t channels, int32_t height, int32_t width, const float* render, int64_t sc, int64_t sy, int64_t sx,
                        int32_t n_appearances, int32_t n_params, const float* exposure_params, const int64_t* appearance_id,
                        int64_t host_appearance_id, int32_t s, const float* shade, float max_gray_scale, float max_gamma,
                        void* workspace, size_t workspace_bytes, const float* v_out, float* v_render, float* v_params, float* v_shade,
                        void* stream) {
    if (int rc = check_exposure(__func__, channels, height, width, render, sc, sy, sx, n_appearances, n_params, exposure_params, s, shade,
                                workspace, workspace_bytes, true, v_out))
        return rc;
    B200GS_CHECK_ARG(v_render && v_params && (s == 0 || v_shade), "NULL pointer");
    const cudaStream_t st = (cudaStream_t)stream;
    float* ws = static_cast<float*>(workspace);
    const ExpoArgs g = make_args(height, width, sc, sy, sx, n_params, s, max_gray_scale, max_gamma);
    exposure_prep_kernel<<<1, PREP_THREADS, 0, st>>>(n_appearances, n_params, exposure_params, appearance_id, host_appearance_id, s, shade, ws);
    B200GS_LAUNCH_CHECK();
    const int64_t n_blocks = pixel_blocks(height, width);
    float* partials = ws + HEAD + s * s;
    float* v_m = s > 0 ? partials + n_blocks * PARTIAL : nullptr;
    const dim3 grid(div_up(width, BX), div_up(height, BY)), block(BX, BY);
    if (s > 0) exposure_bwd_kernel<true><<<grid, block, 0, st>>>(g, render, v_out, ws, v_render, partials, v_m);
    else exposure_bwd_kernel<false><<<grid, block, 0, st>>>(g, render, v_out, ws, v_render, partials, v_m);
    B200GS_LAUNCH_CHECK();
    exposure_reduce_kernel<<<1 + div_up(s * s, RED_THREADS / 32), RED_THREADS, 0, st>>>(g, int(n_blocks), n_appearances, ws, partials, v_m,
                                                                                         shade, v_params, v_shade);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

}  // extern "C"
