// K9/K10: fused L1 + SSIM training loss on the rendered image, the op that follows the rasterizer every step (SURVEY §8f row 2;
// validated against the oracle and the reference-generated golden vectors: tests/test_gpu_loss.py):
//     loss = (1 - lambda) * mean|img - gt| + lambda * (1 - mean(SSIM(img, gt)))          internal/metrics/vanilla_metrics.py:57-74
//     SSIM: 11-tap Gaussian window (sigma 1.5), zero padding, C1 = 0.01^2, C2 = 0.03^2     internal/utils/ssim.py:23-63
// The window is separable; the tile engine is ssim.cuh.  K9 (forward): one CTA per 16x16 tile and channel loads the tile +
// 5-pixel halo of both images into shared memory, blurs the five moments (a, b, a^2, b^2, ab) horizontally then vertically,
// evaluates the SSIM map and writes (i) per-CTA partial sums of |a-b| and SSIM (summed by the caller: deterministic) and (ii)
// the three partial derivative maps d ssim / d(mu_a), d(E[a^2]), d(E[ab]).  K10 (backward): the image cotangent is the same
// blur applied to those maps (the window is symmetric),
//     v_img = w * ( (1-l) sign(a-b) - l * (blur(dmu) + 2 a blur(de11) + b blur(de12)) ) / (C H W).
// Oracle: oracle/loss_oracle.py, pinned to the reference's ssim.py by tests/test_loss_oracle_golden.py.
#include "ssim.cuh"

namespace b200gs {

namespace {

__global__ void __launch_bounds__(LT * LT) loss_fwd_kernel(int width, int height, const float* __restrict__ img, const float* __restrict__ gt,
                                                           float* __restrict__ dmaps, float* __restrict__ partials) {
    __shared__ float s_a[LE][LE], s_b[LE][LE];
    __shared__ float s_h[5][LE][LT];        // horizontally blurred moments: rows with halo, columns of the tile
    __shared__ float s_red[LT * LT / 32][2];
    const int c = blockIdx.z;
    const int x0 = blockIdx.x * LT, y0 = blockIdx.y * LT;
    const int64_t plane = int64_t(width) * height;
    const float* img_c = img + c * plane;
    const float* gt_c = gt + c * plane;
    load_halo(width, height, x0, y0, {s_a}, [=](int, int64_t p) { return __ldg(img_c + p); });
    load_halo(width, height, x0, y0, {s_b}, [=](int, int64_t p) { return __ldg(gt_c + p); });
    __syncthreads();
    blur_moments_h(c_ssim_win, s_a, s_b, s_h);
    __syncthreads();
    const int lx = threadIdx.x % LT, ly = threadIdx.x / LT;
    const int x = x0 + lx, y = y0 + ly;
    const bool inside = x < width && y < height;
    float m[5];
    blur_moments_v(c_ssim_win, s_h, ly, lx, m);
    float acc[2] = {0.f, 0.f};              // |a - b|, SSIM
    if (inside) {
        const float a = s_a[ly + HALO][lx + HALO], b = s_b[ly + HALO][lx + HALO];
        const SsimTerms t = ssim_terms<0>(m, SSIM_C1, SSIM_C2);
        acc[0] = fabsf(a - b);
        acc[1] = t.ssim;
        const int64_t p = c * plane + int64_t(y) * width + x;
        const int64_t stride = int64_t(gridDim.z) * plane;
        dmaps[p] = t.d_mu;
        dmaps[stride + p] = t.d_xx;
        dmaps[2 * stride + p] = t.d_ab;
    }
    // per-CTA partial sums (summed by the caller in a fixed order)
    cta_sum_row(acc, s_red, threadIdx.x,
                [&] { return partials + 2 * ((int64_t(blockIdx.z) * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x); });
}

__global__ void __launch_bounds__(LT * LT) loss_bwd_kernel(int width, int height, const float* __restrict__ img, const float* __restrict__ gt,
                                                           const float* __restrict__ dmaps, float lambda, const float* __restrict__ v_loss,
                                                           float* __restrict__ v_img) {
    __shared__ float s_m[3][LE][LE];
    __shared__ float s_h[3][LE][LT];
    const int c = blockIdx.z;
    const int x0 = blockIdx.x * LT, y0 = blockIdx.y * LT;
    const int64_t plane = int64_t(width) * height;
    const int64_t stride = int64_t(gridDim.z) * plane;
#pragma unroll
    for (int m = 0; m < 3; ++m) {
        const float* map = dmaps + m * stride + c * plane;
        load_halo(width, height, x0, y0, {s_m[m]}, [=](int, int64_t p) { return __ldg(map + p); });
    }
    __syncthreads();
    blur_maps_h(c_ssim_win, s_m, s_h);
    __syncthreads();
    const int lx = threadIdx.x % LT, ly = threadIdx.x / LT;
    const int x = x0 + lx, y = y0 + ly;
    if (x >= width || y >= height) return;
    float g[3];
    blur_maps_v(c_ssim_win, s_h, ly, lx, g);
    const int64_t p = c * plane + int64_t(y) * width + x;
    const float a = __ldg(img + p), b = __ldg(gt + p);
    const float d = a - b;
    const float sgn = d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f);          // torch.abs' subgradient at 0 is 0
    const float inv_n = 1.f / (float(gridDim.z) * float(width) * float(height));
    const float up = v_loss ? __ldg(v_loss) : 1.f;
    v_img[p] = up * inv_n * ((1.f - lambda) * sgn - lambda * ssim_grad(g, a, b));
}

// the grid is (ceil(W/LT), ceil(H/LT), C): C and ceil(H/LT) are at most 65535, and ceil(W/LT) is computed in int
bool loss_size_ok(int32_t channels, int32_t width, int32_t height) {
    return channels >= 1 && width >= 1 && height >= 1 && channels <= 65535 && height <= 65535 * LT && width <= INT32_MAX - (LT - 1);
}

// shared by the forward and the backward; returns the error code, or 0 when the arguments are valid
int check_loss(const char* fn, int32_t channels, int32_t width, int32_t height, const void* image, const void* target, const void* maps,
               const void* out) {
    if (channels < 1 || width < 1 || height < 1) return fail(fn, "bad size: channels, width and height must be >= 1");
    if (channels > 65535) return fail(fn, "too many channels (> 65535)");
    if (height > 65535 * LT) return fail(fn, "image too tall (height > 65535 * 16)");
    if (width > INT32_MAX - (LT - 1)) return fail(fn, "image too wide (width > 2^31 - 16)");
    if (!(image && target && maps && out)) return fail(fn, "NULL pointer");
    return 0;
}

}  // namespace

}  // namespace b200gs

using namespace b200gs;

extern "C" {

int64_t b200gs_loss_blocks(int32_t channels, int32_t width, int32_t height) {
    return loss_size_ok(channels, width, height) ? int64_t(channels) * div_up(width, LT) * div_up(height, LT) : 0;
}

int b200gs_loss_fwd(int32_t channels, int32_t width, int32_t height, const float* image, const float* target, float* dmaps,
                    float* partials, void* stream) {
    if (int rc = check_loss(__func__, channels, width, height, image, target, dmaps, partials)) return rc;
    const dim3 grid(div_up(width, LT), div_up(height, LT), channels);
    loss_fwd_kernel<<<grid, LT * LT, 0, (cudaStream_t)stream>>>(width, height, image, target, dmaps, partials);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

int b200gs_loss_bwd(int32_t channels, int32_t width, int32_t height, const float* image, const float* target, const float* dmaps,
                    float lambda_dssim, const float* v_loss, float* v_image, void* stream) {
    if (int rc = check_loss(__func__, channels, width, height, image, target, dmaps, v_image)) return rc;
    const dim3 grid(div_up(width, LT), div_up(height, LT), channels);
    loss_bwd_kernel<<<grid, LT * LT, 0, (cudaStream_t)stream>>>(width, height, image, target, dmaps, lambda_dssim, v_loss, v_image);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

}  // extern "C"
