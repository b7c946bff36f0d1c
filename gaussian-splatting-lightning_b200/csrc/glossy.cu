// K47 / K48: Glossy-Gaussian view-dependent opacity and SH colour of every Gaussian, forward and backward, one thread per Gaussian.
//
// Restates GlossyRendererModule.get_opacities / get_rgbs (internal/renderers/glossy_renderer.py) with
// GlossyGaussianModel.get_view_dep_opacities (internal/models/glossy_gaussian.py:66-79, eval_sh_decomposed of sh_utils.py:115-171):
//   dir     = (means - campos) / max(|means - campos|, 1e-12)                     (F.normalize; detached: no means gradient)
//   opacity = clamp(SH_deg(op_dc | op_rest; dir) + 0.5, 0, 1)                    every row (the reference ignores the masks here)
//   rgb     = clamp(SH_deg(shs; dir) + 0.5, min=0)  on mask rows,  0.5 elsewhere  (gsplat's masked SH, then the clamp)
// The basis, the coefficient loader and the staged gradient-row stores are K1 / K8 / K15's (sh.cuh).
//
// HBM-bound: per Gaussian at degree 3 with 16-coefficient colour and opacity storage, 286 B forward (means 12, opacity 4 + 60,
// colour 12 + 180, mask 1 in; opacity 4, rgb 12, clamp bits 1 out) and 285 B backward (means 12, clamp bits 1, cotangents 4 + 12
// in; opacity gradient 4 + 60, colour gradient 12 + 180 out).  The backward reads no coefficient: the forward's clamp bits carry
// every decision it needs.
#include "common.cuh"
#include "sh.cuh"

namespace b200gs {

namespace {

constexpr int GLOSSY_FWD_THREADS = 256;
constexpr int GLOSSY_BWD_THREADS = 128;

// Clamp bits of one Gaussian, K47 -> K48.  A set bit stops that output's gradient: torch.clamp passes the gradient where
// min <= x <= max (bounds inclusive), so a bit is set where that test fails, NaN included.  A masked row sets all three colour
// bits (its coefficients get no gradient).
constexpr uint8_t GLOSSY_RGB_BITS = 7;     // bit c: channel c of the colour
constexpr uint8_t GLOSSY_OPACITY_BIT = 8;

__device__ __forceinline__ float unit_dir_to(const float* __restrict__ means, const float* __restrict__ campos, int64_t i, float& dx,
                                             float& dy, float& dz) {
    dx = __ldg(means + 3 * i) - __ldg(campos);
    dy = __ldg(means + 3 * i + 1) - __ldg(campos + 1);
    dz = __ldg(means + 3 * i + 2) - __ldg(campos + 2);
    return normalize_dir(dx, dy, dz);
}

// SPLIT: colour = dc shs [n,1,3] | rest shs_rest [n,sh_stride-1,3]; otherwise shs [n,sh_stride,3].  rgb NULL: no colour.
template <bool SPLIT, int MC>
__global__ void __launch_bounds__(GLOSSY_FWD_THREADS) glossy_fwd_kernel(int deg, int64_t n, const float* __restrict__ means,
                                                                        const float* __restrict__ campos, const float* __restrict__ op_dc,
                                                                        const float* __restrict__ op_rest, int op_k_rest,
                                                                        const float* __restrict__ shs, const float* __restrict__ shs_rest,
                                                                        int sh_stride, const uint8_t* __restrict__ mask,
                                                                        float* __restrict__ opacity, float* __restrict__ rgb,
                                                                        uint8_t* __restrict__ clamped) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int ncoef = (deg + 1) * (deg + 1);
    float dx, dy, dz;
    unit_dir_to(means, campos, i, dx, dy, dz);
    float bs[MC];
    sh_basis<MC>(deg, dx, dy, dz, bs);

    const float* orow = op_rest + i * int64_t(op_k_rest);
    float o = bs[0] * __ldg(op_dc + i);
#pragma unroll
    for (int k = 1; k < MC; ++k)
        if (k < ncoef) o += bs[k] * __ldg(orow + k - 1);
    o += 0.5f;
    uint8_t cl = (o >= 0.f && o <= 1.f) ? 0 : GLOSSY_OPACITY_BIT;
    opacity[i] = o < 0.f ? 0.f : (o > 1.f ? 1.f : o);       // NaN stays NaN, as in torch.clamp

    if (rgb != nullptr) {
        float c[3] = {0.5f, 0.5f, 0.5f};
        if (mask != nullptr && __ldg(mask + i) == 0) {
            cl |= GLOSSY_RGB_BITS;
        } else {
            float sh[MC * 3];
            load_sh_any<SPLIT, MC>(shs, shs_rest, i, sh_stride, ncoef, sh);
            float r = 0.f, g = 0.f, b = 0.f;
#pragma unroll
            for (int k = 0; k < MC; ++k)
                if (k < ncoef) { r += bs[k] * sh[3 * k]; g += bs[k] * sh[3 * k + 1]; b += bs[k] * sh[3 * k + 2]; }
            c[0] = r + 0.5f; c[1] = g + 0.5f; c[2] = b + 0.5f;
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                if (!(c[j] >= 0.f)) cl |= uint8_t(1u << j);
                c[j] = c[j] < 0.f ? 0.f : c[j];
            }
        }
        rgb[3 * i] = c[0]; rgb[3 * i + 1] = c[1]; rgb[3 * i + 2] = c[2];
    }
    clamped[i] = cl;
}

// One gradient row of width rw: coefficient k (k0 <= k < MC) at columns (k - k0) * CH .. + CH - 1 gets basis_k * g[channel] below
// the active degree and 0 at or beyond it; columns past the kernel's MC coefficients get 0.
template <int MC, int CH>
__device__ __forceinline__ void fill_grad_row(float* row, int rw, int k0, int ncoef, const float* bs, const float* g) {
#pragma unroll
    for (int k = 0; k < MC; ++k) {
        const int c = (k - k0) * CH;
        if (k >= k0 && c < rw) {
            const float bk = k < ncoef ? bs[k] : 0.f;
#pragma unroll
            for (int j = 0; j < CH; ++j) row[c + j] = bk * g[j];
        }
    }
    for (int c = (MC - k0) * CH; c < rw; ++c) row[c] = 0.f;
}

// Writes the gradient rows of the warp's 32 Gaussians: staged and flushed coalesced when a row fits the staging buffer (rw is
// warp-uniform), otherwise one row per thread.  Every lane of the warp must call it.
template <int MC, int CH>
__device__ __forceinline__ void store_grad_rows(float* s_warp, unsigned lane, int64_t i, int64_t n, float* __restrict__ dst, int rw, int k0,
                                                int ncoef, const float* bs, const float* g) {
    if (rw == 0) return;
    if (rw <= MC * 3) {
        fill_grad_row<MC, CH>(s_warp + lane * (rw | 1), rw, k0, ncoef, bs, g);
        flush_sh_rows(s_warp, rw, i, n, lane, dst, false);
        __syncwarp();                                   // the next row reuses the staging buffer
    } else if (i < n) {
        fill_grad_row<MC, CH>(dst + i * int64_t(rw), rw, k0, ncoef, bs, g);
    }
}

// v_rgb NULL: no colour gradient (v_shs / v_shs_rest not written).  Every other output row is written in full.
template <bool SPLIT, int MC>
__global__ void __launch_bounds__(GLOSSY_BWD_THREADS) glossy_bwd_kernel(int deg, int64_t n, const float* __restrict__ means,
                                                                        const float* __restrict__ campos, int op_k_rest, int sh_stride,
                                                                        const uint8_t* __restrict__ clamped,
                                                                        const float* __restrict__ v_opacity, const float* __restrict__ v_rgb,
                                                                        float* __restrict__ v_op_dc, float* __restrict__ v_op_rest,
                                                                        float* __restrict__ v_shs, float* __restrict__ v_shs_rest) {
    __shared__ float s_rows[GLOSSY_BWD_THREADS / 32][32 * (MC * 3 + 1)];
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    const unsigned lane = threadIdx.x & 31u;
    float* s_warp = s_rows[threadIdx.x >> 5];
    const bool in_range = i < n;
    const int ncoef = (deg + 1) * (deg + 1);
    float bs[MC];
#pragma unroll
    for (int k = 0; k < MC; ++k) bs[k] = 0.f;
    uint8_t cl = 0;
    float go = 0.f;
    if (in_range) {
        float dx, dy, dz;
        unit_dir_to(means, campos, i, dx, dy, dz);
        sh_basis<MC>(deg, dx, dy, dz, bs);
        cl = __ldg(clamped + i);
        go = (cl & GLOSSY_OPACITY_BIT) ? 0.f : __ldg(v_opacity + i);
        v_op_dc[i] = bs[0] * go;
    }
    store_grad_rows<MC, 1>(s_warp, lane, i, n, v_op_rest, op_k_rest, 1, ncoef, bs, &go);
    if (v_rgb == nullptr) return;     // uniform over the grid
    float g[3] = {0.f, 0.f, 0.f};
    if (in_range) {
#pragma unroll
        for (int j = 0; j < 3; ++j) g[j] = ((cl >> j) & 1) ? 0.f : __ldg(v_rgb + 3 * i + j);
        if (SPLIT) { v_shs[3 * i] = bs[0] * g[0]; v_shs[3 * i + 1] = bs[0] * g[1]; v_shs[3 * i + 2] = bs[0] * g[2]; }
    }
    if (SPLIT)
        store_grad_rows<MC, 3>(s_warp, lane, i, n, v_shs_rest, (sh_stride - 1) * 3, 1, ncoef, bs, g);
    else
        store_grad_rows<MC, 3>(s_warp, lane, i, n, v_shs, sh_stride * 3, 0, ncoef, bs, g);
}

// shared by the Glossy-Gaussian entry points: the degree, the opacity rest width and, when the colour is on, its layout
int check_glossy(const char* fn, int32_t degree, int64_t n, const float* means, const float* campos, int32_t op_k_rest, bool colour,
                 int32_t sh_stride, int32_t sh_split) {
    if (degree < 0 || degree > 4) return fail(fn, "degree must be 0..4");
    if (n < 0) return fail(fn, "n < 0");
    if (op_k_rest < 0 || op_k_rest + 1 < (degree + 1) * (degree + 1)) return fail(fn, "1 + op_k_rest < (degree+1)^2");
    if (n > 0 && !(means && campos)) return fail(fn, "NULL pointer");
    if (colour && sh_split != 0 && sh_split != 1) return fail(fn, "sh_split must be 0 or 1");
    if (colour && sh_stride < (degree + 1) * (degree + 1)) return fail(fn, "sh_stride < (degree+1)^2");
    return 0;
}

}  // namespace

}  // namespace b200gs

using namespace b200gs;

extern "C" {

// The instantiation is picked here, by the degree (MC = 25 iff degree 4) and the colour layout.
int b200gs_glossy_sh_fwd(int32_t degree, int64_t n, const float* means, const float* campos, const float* op_dc, const float* op_rest,
                         int32_t op_k_rest, const float* shs, const float* shs_rest, int32_t sh_stride, int32_t sh_split,
                         const uint8_t* mask, float* opacity, float* rgb, uint8_t* clamped, void* stream) {
    if (int rc = check_glossy(__func__, degree, n, means, campos, op_k_rest, rgb != nullptr, sh_stride, sh_split)) return rc;
    B200GS_CHECK_ARG(n == 0 || (op_dc && opacity && clamped && (op_k_rest == 0 || op_rest)), "NULL pointer");
    B200GS_CHECK_ARG(n == 0 || !rgb || (shs && (!sh_split || sh_stride == 1 || shs_rest)), "NULL pointer");
    static constexpr decltype(&glossy_fwd_kernel<false, 16>) kernels[2][2] = {
        {glossy_fwd_kernel<false, 16>, glossy_fwd_kernel<false, 25>}, {glossy_fwd_kernel<true, 16>, glossy_fwd_kernel<true, 25>}};
    if (n == 0) return B200GS_OK;
    kernels[sh_split != 0][degree > 3]<<<(unsigned)div_up64(n, GLOSSY_FWD_THREADS), GLOSSY_FWD_THREADS, 0, (cudaStream_t)stream>>>(
        degree, n, means, campos, op_dc, op_rest, op_k_rest, shs, shs_rest, sh_stride, mask, opacity, rgb, clamped);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

int b200gs_glossy_sh_bwd(int32_t degree, int64_t n, const float* means, const float* campos, int32_t op_k_rest, int32_t sh_stride,
                         int32_t sh_split, const uint8_t* clamped, const float* v_opacity, const float* v_rgb, float* v_op_dc,
                         float* v_op_rest, float* v_shs, float* v_shs_rest, void* stream) {
    if (int rc = check_glossy(__func__, degree, n, means, campos, op_k_rest, v_rgb != nullptr, sh_stride, sh_split)) return rc;
    B200GS_CHECK_ARG(n == 0 || (clamped && v_opacity && v_op_dc && (op_k_rest == 0 || v_op_rest)), "NULL pointer");
    B200GS_CHECK_ARG(n == 0 || !v_rgb || (v_shs && (!sh_split || sh_stride == 1 || v_shs_rest)), "NULL pointer");
    static constexpr decltype(&glossy_bwd_kernel<false, 16>) kernels[2][2] = {
        {glossy_bwd_kernel<false, 16>, glossy_bwd_kernel<false, 25>}, {glossy_bwd_kernel<true, 16>, glossy_bwd_kernel<true, 25>}};
    if (n == 0) return B200GS_OK;
    kernels[sh_split != 0][degree > 3]<<<(unsigned)div_up64(n, GLOSSY_BWD_THREADS), GLOSSY_BWD_THREADS, 0, (cudaStream_t)stream>>>(
        degree, n, means, campos, op_k_rest, sh_stride, clamped, v_opacity, v_rgb, v_op_dc, v_op_rest, v_shs, v_shs_rest);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

}  // extern "C"
