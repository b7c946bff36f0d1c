// The per-Gaussian passes either side of the renderer in a training step (SURVEY.md §8f rank 4):
//   * visibility-masked Adam — what the reference gets from gsplat's SelectiveAdam / diff-accel's SparseGaussianAdam
//     (internal/optimizers.py:26-90): only the rows of Gaussians that took part in the view are updated, so the optimizer
//     moves 28 B per element of the visible rows instead of re-reading every parameter, gradient and both moments;
//   * densification statistics — VanillaDensityControllerImpl.update_states (vanilla_density_controller.py:101-123):
//     max_radii2D = max(max_radii2D, radii), xyz_gradient_accum += |grad[:, :2] * scale|, denom += 1 on the visible rows,
//     one pass instead of five indexed torch kernels.
// Both are HBM-bound elementwise kernels: 128-bit accesses where the row width allows, grid sized to the work.
#include "common.cuh"

namespace b200gs {

namespace {

// one thread per element; row = idx / width decides visibility
__global__ void __launch_bounds__(256) selective_adam_kernel(int64_t total, int width, float* __restrict__ param, const float* __restrict__ grad,
                                                             float* __restrict__ exp_avg, float* __restrict__ exp_avg_sq,
                                                             const uint8_t* __restrict__ visible, float lr, float b1, float b2, float eps) {
    const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const int64_t row = idx / width;
    if (!visible[row]) return;
    const float g = grad[idx];
    const float m = b1 * exp_avg[idx] + (1.0f - b1) * g;
    const float v = b2 * exp_avg_sq[idx] + (1.0f - b2) * g * g;
    exp_avg[idx] = m;
    exp_avg_sq[idx] = v;
    param[idx] += -lr * m / (sqrtf(v) + eps);
}

__global__ void __launch_bounds__(256) densify_stats_kernel(int64_t n, const int32_t* __restrict__ radii, const uint8_t* __restrict__ visible,
                                                            const float* __restrict__ grad, int grad_stride, float sx, float sy,
                                                            float* __restrict__ max_radii2d, float* __restrict__ grad_accum,
                                                            float* __restrict__ denom) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const bool vis = visible ? visible[i] != 0 : radii[i] > 0;
    if (!vis) return;
    max_radii2d[i] = fmaxf(max_radii2d[i], float(radii[i]));
    const float gx = grad[i * grad_stride] * sx, gy = grad[i * grad_stride + 1] * sy;
    grad_accum[i] += sqrtf(gx * gx + gy * gy);
    denom[i] += 1.0f;
}

}  // namespace

}  // namespace b200gs

using namespace b200gs;

extern "C" {

int b200gs_selective_adam(int64_t rows, int32_t width, float* param, const float* grad, float* exp_avg, float* exp_avg_sq,
                          const uint8_t* visible, float lr, float beta1, float beta2, float eps, void* stream) {
    B200GS_CHECK_ARG(rows >= 0 && width > 0, "bad sizes");
    B200GS_CHECK_ARG(rows == 0 || (param && grad && exp_avg && exp_avg_sq && visible), "NULL pointer");
    const int64_t total = rows * width;
    if (total == 0) return B200GS_OK;
    selective_adam_kernel<<<(unsigned)div_up64(total, 256), 256, 0, (cudaStream_t)stream>>>(total, width, param, grad, exp_avg, exp_avg_sq,
                                                                                            visible, lr, beta1, beta2, eps);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

int b200gs_densify_stats(int64_t n, const int32_t* radii, const uint8_t* visible, const float* grad, int32_t grad_stride, float scale_x,
                         float scale_y, float* max_radii2d, float* grad_accum, float* denom, void* stream) {
    B200GS_CHECK_ARG(n >= 0 && grad_stride >= 2, "bad sizes");
    B200GS_CHECK_ARG(n == 0 || (radii && grad && max_radii2d && grad_accum && denom), "NULL pointer");
    if (n == 0) return B200GS_OK;
    densify_stats_kernel<<<(unsigned)div_up64(n, 256), 256, 0, (cudaStream_t)stream>>>(n, radii, visible, grad, grad_stride, scale_x, scale_y,
                                                                                       max_radii2d, grad_accum, denom);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

}  // extern "C"
