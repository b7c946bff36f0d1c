// The two per-Gaussian passes of 3DGS-MCMC training (internal/density_controllers/mcmc_density_controller.py):
//   * relocation — gsplat's compute_relocation (Eq. (9) of the paper), the opacity / scale of a Gaussian that N samples now share;
//   * position noise — _add_xyz_noise, the per-step SGLD perturbation of the means shaped by each Gaussian's covariance.
// Both are elementwise.  The noise pass runs after every training step over all N Gaussians and is HBM-bound (44 B read,
// 12 B written per Gaussian); relocation runs on the few Gaussians sampled every 100 steps.
#include <curand_kernel.h>

#include "common.cuh"
#include "geometry.cuh"

namespace b200gs {

namespace {

// D = sum_{j=1..N} (-1)^(j-1) C(N,j) o'^j / sqrt(j).  The alternating terms reach (1 + o')^N (<= e^16.6 for fp32 opacities), so
// the sum is taken in fp64 with the term C(N,j) o'^j carried by the recurrence a_j = a_{j-1} o' (N-j+1) / j.
__global__ void __launch_bounds__(256) relocation_kernel(int64_t n, const float* __restrict__ opacities, const float* __restrict__ scales,
                                                         const int32_t* __restrict__ counts, int n_max, float* __restrict__ new_opacities,
                                                         float* __restrict__ new_scales) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int N = min(max(counts[i], 1), n_max);
    const double o = opacities[i];
    const double op = -expm1(log1p(-o) / N);     // 1 - (1 - o)^(1/N) without cancellation as o -> 1
    double a = 1.0, D = 0.0;
    for (int j = 1; j <= N; ++j) {
        a = a * op * double(N - j + 1) / double(j);
        const double t = a / sqrt(double(j));
        D += (j & 1) ? t : -t;
    }
    const double coef = o / D;
    new_opacities[i] = float(op);
#pragma unroll
    for (int k = 0; k < 3; ++k) new_scales[3 * i + k] = float(coef * double(scales[3 * i + k]));
}

// The covariance comes from the rasterizer's own code (load_scale_quat<RAW> + gaussian_cov3d, in fp32 as in K8: the noise is a random
// step, and fp32 puts ~1e-6 relative on it); z from Philox4x32-10 keyed by (seed, subsequence offset + i), so a Gaussian's draw does
// not depend on the launch shape.  Every load is issued before the arithmetic.
__global__ void __launch_bounds__(256) position_noise_kernel(int64_t n, float* __restrict__ means, const float* __restrict__ log_scales,
                                                             const float* __restrict__ raw_quats, const float* __restrict__ opacity_logits,
                                                             float scale, uint64_t seed, uint64_t offset) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float p0 = means[3 * i], p1 = means[3 * i + 1], p2 = means[3 * i + 2];
    const float logit = __ldg(opacity_logits + i);
    float sc[3], q[4], inv_qn;
    load_scale_quat<true, float>(log_scales, raw_quats, i, sc, q, &inv_qn);
    Proj<float> g;
    gaussian_cov3d<float>(sc, q, 1.0f, g);
    const float o = 1.0f / (1.0f + expf(-logit));
    const float w = 1.0f / (1.0f + expf(-100.0f * ((1.0f - o) - 0.995f)));   // op_sigmoid(1 - o); exactly 0 once exp overflows (o > 0.89)
    curandStatePhilox4_32_10_t st;
    curand_init(seed, offset + uint64_t(i), 0, &st);
    const float4 z = curand_normal4(&st);
    const float c = scale * w;
    const float* S = g.S3;   // xx xy xz yy yz zz
    means[3 * i] = p0 + c * (S[0] * z.x + S[1] * z.y + S[2] * z.z);
    means[3 * i + 1] = p1 + c * (S[1] * z.x + S[3] * z.y + S[4] * z.z);
    means[3 * i + 2] = p2 + c * (S[2] * z.x + S[4] * z.y + S[5] * z.z);
}

}  // namespace

}  // namespace b200gs

using namespace b200gs;

extern "C" {

int b200gs_mcmc_relocation(int64_t n, const float* opacities, const float* scales, const int32_t* counts, const float* binoms, int32_t n_max,
                           float* new_opacities, float* new_scales, void* stream) {
    B200GS_CHECK_ARG(n >= 0, "n < 0");
    B200GS_CHECK_ARG(n_max >= 1, "n_max < 1");
    B200GS_CHECK_ARG(n == 0 || (opacities && scales && counts && binoms && new_opacities && new_scales), "NULL pointer");
    if (n == 0) return B200GS_OK;
    relocation_kernel<<<(unsigned)div_up64(n, 256), 256, 0, (cudaStream_t)stream>>>(n, opacities, scales, counts, n_max, new_opacities,
                                                                                    new_scales);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

int b200gs_mcmc_position_noise(int64_t n, float* means, const float* log_scales, const float* raw_quats, const float* opacity_logits,
                               float scale, uint64_t seed, uint64_t offset, void* stream) {
    B200GS_CHECK_ARG(n >= 0, "n < 0");
    B200GS_CHECK_ARG(n == 0 || (means && log_scales && raw_quats && opacity_logits), "NULL pointer");
    B200GS_CHECK_ARG((reinterpret_cast<uintptr_t>(raw_quats) & 15u) == 0, "raw_quats must be 16-byte aligned");
    if (n == 0) return B200GS_OK;
    position_noise_kernel<<<(unsigned)div_up64(n, 256), 256, 0, (cudaStream_t)stream>>>(n, means, log_scales, raw_quats, opacity_logits, scale,
                                                                                        seed, offset);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

}  // extern "C"
