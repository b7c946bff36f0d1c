// K27-K31: inverse-depth regularisation loss, HasInverseDepthMetricsModule.get_inverse_depth_metric
// (internal/metrics/inverse_depth_metrics.py:70-107), on pred and gt [H,W] with an optional 0/1 keep-mask:
//     pred' = (pred - min) / (max - min + 1e-8)   (norm 1, min/max of the whole pred, constants)
//           | pred / median                      (norm 2)
//           | pred / mean(gt), gt' = gt / mean(gt) (norm 3)
//     a = gt' k, b = pred' k                      (k the keep-mask, 1 without one)
//     l1: mean|a - b|   l2: mean (a - b)^2   l1+ssim: (1 - w) l1 + w (1 - SSIM_tm(a, b))
// SSIM_tm is torchmetrics' SSIM with its defaults (11-tap Gaussian, sigma 1.5, k1 0.01, k2 0.03), whose data range is
// dr = max(range(a), range(b)) and C1 = (0.01 dr)^2, C2 = (0.03 dr)^2.  Its reflect pad followed by the 5-pixel crop keeps exactly
// the windows that lie inside the image, so SSIM is the mean over the (H-10)(W-10) full-window positions.  The gradient flows
// through dr into b's extremum pixels, split evenly among tied pixels (torch's max()/min()), and half of it on a tie of the two
// ranges (torch.max(a, b)).
//   * K27 stats: per-CTA partials of min/max of pred and gt and of the sum of gt (one empty CTA when nothing uses them).
//   * K28 prep (one CTA): adds them in block order and writes the normalisation constants, b's extrema, dr, C1 and C2 to the
//     workspace head.  Normalisations are positive and monotone in float32, so b's extrema are those of pred, normalised.
//   * K29 fwd: 16x16 tiles; per-CTA partials of |a-b| or (a-b)^2 and, with SSIM, of the SSIM map, its derivatives with C1 and
//     C2, and the number of pixels tied at b's max and min; with SSIM also the three derivative maps of the map with b's blurred
//     moments (mu_b, E[b^2], E[ab]), zero outside the full-window positions.  K29 and K31 run the SSIM tile engine of ssim.cuh
//     with torchmetrics' window, differentiated in b.
//   * K30 loss (one CTA): adds the partials in block order, writes the loss, the statistics and the backward's coefficients.
//   * K31 bwd: v_pred = up * chain * (L1/L2 term + blur of the maps + the dr term at the extremum pixels).
// No float atomics: every sum has a fixed order, so two backwards are bit-identical.
#include "ssim.cuh"

namespace b200gs {

namespace {

constexpr int STAT_THREADS = 256;
constexpr int STAT_PIXELS = 2048;       // pixels per stats CTA before the grid saturates
constexpr int STAT_MAX_BLOCKS = 1024;
constexpr int RED_THREADS = 1024;
constexpr int STAT = 8;                 // floats per stats partial: pred min, max, gt min, max, gt sum
constexpr int PART = 8;                 // floats per tile partial: sum l, sum ssim, sum dssim/dC1, dC2, n at b max, n at b min
constexpr int HEAD = 16;
enum Head { H_SUB, H_DIV, H_BMAX, H_BMIN, H_C1, H_C2, H_DR, H_SHARE, H_GMAX, H_GMIN, H_VL, H_VS };

// torchmetrics' float32 Gaussian: exp(-(d / 1.5)^2 / 2) over d = -5..5, divided by its float32 sum
__device__ __constant__ float c_win[TAPS] = {1.028380357e-03f, 7.598755881e-03f, 3.600077331e-02f, 1.093606800e-01f, 2.130055279e-01f,
                                             2.660117149e-01f, 2.130055279e-01f, 1.093606800e-01f, 3.600077331e-02f, 7.598755881e-03f,
                                             1.028380357e-03f};

struct DArgs {
    int height, width;
    int l2, norm;
    int64_t msy, msx;                   // keep-mask element strides
    float median, w;
};

// correctly rounded divisions (the library builds with --use_fast_math), so the normalisation is monotone and b's extrema are
// those of pred, normalised
__device__ __forceinline__ float norm_pred(float p, int norm, float sub, float div) {
    switch (norm) {
    case 1: return __fdiv_rn(p - sub, div);
    case 2: return p * div;             // torch divides by a CPU scalar as a product with its float reciprocal
    case 3: return __fdiv_rn(p, div);
    default: return p;
    }
}

__device__ __forceinline__ float norm_gt(float g, int norm, float div) { return norm == 3 ? __fdiv_rn(g, div) : g; }

__device__ __forceinline__ bool kept(const uint8_t* __restrict__ mask, const DArgs& g, int y, int x) {
    return mask == nullptr || __ldg(mask + g.msy * y + g.msx * x) != 0;
}

__global__ void __launch_bounds__(STAT_THREADS) depth_stats_kernel(int64_t n, const float* __restrict__ pred, const float* __restrict__ gt,
                                                                   float* __restrict__ partials) {
    __shared__ float s[STAT_THREADS / 32][5];
    float v[5] = {INFINITY, -INFINITY, INFINITY, -INFINITY, 0.f};
    for (int64_t i = int64_t(blockIdx.x) * STAT_THREADS + threadIdx.x; i < n; i += int64_t(gridDim.x) * STAT_THREADS) {
        const float p = __ldg(pred + i), q = __ldg(gt + i);
        v[0] = fminf(v[0], p); v[1] = fmaxf(v[1], p);
        v[2] = fminf(v[2], q); v[3] = fmaxf(v[3], q);
        v[4] += q;
    }
    v[0] = warp_reduce<Min>(v[0]); v[1] = warp_reduce<Max>(v[1]); v[2] = warp_reduce<Min>(v[2]); v[3] = warp_reduce<Max>(v[3]);
    v[4] = warp_sum(v[4]);
    const int warp = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int k = 0; k < 5; ++k) s[warp][k] = v[k];
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < STAT_THREADS / 32; ++w) {
            v[0] = fminf(v[0], s[w][0]); v[1] = fmaxf(v[1], s[w][1]);
            v[2] = fminf(v[2], s[w][2]); v[3] = fmaxf(v[3], s[w][3]);
            v[4] += s[w][4];
        }
#pragma unroll
        for (int k = 0; k < 5; ++k) partials[int64_t(blockIdx.x) * STAT + k] = v[k];
    }
}

__global__ void __launch_bounds__(RED_THREADS) depth_prep_kernel(DArgs g, int n_blocks, const float* __restrict__ partials,
                                                                 float* __restrict__ head) {
    __shared__ float s_f[RED_THREADS / 32][4];
    __shared__ double s_d[RED_THREADS / 32];
    const int t = threadIdx.x, warp = t >> 5;
    float v[4] = {INFINITY, -INFINITY, INFINITY, -INFINITY};
    double sum = 0.0;
    for (int b = t; b < n_blocks; b += RED_THREADS) {
        const float* p = partials + int64_t(b) * STAT;
        v[0] = fminf(v[0], p[0]); v[1] = fmaxf(v[1], p[1]); v[2] = fminf(v[2], p[2]); v[3] = fmaxf(v[3], p[3]);
        sum += double(p[4]);
    }
    v[0] = warp_reduce<Min>(v[0]); v[1] = warp_reduce<Max>(v[1]); v[2] = warp_reduce<Min>(v[2]); v[3] = warp_reduce<Max>(v[3]);
    sum = warp_reduce<Sum>(sum);
    if ((t & 31) == 0) {
#pragma unroll
        for (int k = 0; k < 4; ++k) s_f[warp][k] = v[k];
        s_d[warp] = sum;
    }
    __syncthreads();
    if (t != 0) return;
    for (int w = 1; w < RED_THREADS / 32; ++w) {
        v[0] = fminf(v[0], s_f[w][0]); v[1] = fmaxf(v[1], s_f[w][1]); v[2] = fminf(v[2], s_f[w][2]); v[3] = fmaxf(v[3], s_f[w][3]);
        sum += s_d[w];
    }
    const float pmin = v[0], pmax = v[1];
    float sub = 0.f, div = 1.f;
    if (g.norm == 1) { sub = pmin; div = (pmax - pmin) + 1e-8f; }
    else if (g.norm == 2) div = __frcp_rn(g.median);
    else if (g.norm == 3) div = float(sum / (double(g.height) * g.width));
    const float bmax = norm_pred(pmax, g.norm, sub, div), bmin = norm_pred(pmin, g.norm, sub, div);
    const float ra = norm_gt(v[3], g.norm, div) - norm_gt(v[2], g.norm, div), rb = bmax - bmin;
    const float dr = fmaxf(ra, rb);
    head[H_SUB] = sub; head[H_DIV] = div; head[H_BMAX] = bmax; head[H_BMIN] = bmin;
    head[H_C1] = (0.01f * dr) * (0.01f * dr);
    head[H_C2] = (0.03f * dr) * (0.03f * dr);
    head[H_DR] = dr;
    head[H_SHARE] = rb > ra ? 1.f : (rb == ra ? 0.5f : 0.f);
}

template <bool SSIM>
__global__ void __launch_bounds__(LT * LT) depth_fwd_kernel(DArgs g, const float* __restrict__ pred, const float* __restrict__ gt,
                                                            const uint8_t* __restrict__ mask, const float* __restrict__ head,
                                                            float* __restrict__ maps, float* __restrict__ partials) {
    __shared__ float s_a[SSIM ? LE : 1][LE], s_b[SSIM ? LE : 1][LE];
    __shared__ float s_h[SSIM ? 5 : 1][LE][LT];
    __shared__ float s_red[LT * LT / 32][6];
    const int x0 = blockIdx.x * LT, y0 = blockIdx.y * LT;
    const int lx = threadIdx.x % LT, ly = threadIdx.x / LT;
    const int x = x0 + lx, y = y0 + ly;
    const bool inside = x < g.width && y < g.height;
    const float sub = __ldg(head + H_SUB), div = __ldg(head + H_DIV);
    float acc[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if constexpr (SSIM) {
        // the halo tiles of a' and b', normalised
        load_halo(g.width, g.height, x0, y0, {s_a, s_b}, [&](int m, int64_t p) {
            return m == 0 ? norm_gt(__ldg(gt + p), g.norm, div) : norm_pred(__ldg(pred + p), g.norm, sub, div);
        });
        __syncthreads();
        blur_moments_h(c_win, s_a, s_b, s_h);
        __syncthreads();
        if (inside) {
            const float a = s_a[ly + HALO][lx + HALO], b = s_b[ly + HALO][lx + HALO];
            acc[0] = fabsf(a - b);
            acc[4] = b == __ldg(head + H_BMAX) ? 1.f : 0.f;
            acc[5] = b == __ldg(head + H_BMIN) ? 1.f : 0.f;
            float d_mu = 0.f, d_bb = 0.f, d_ab = 0.f;
            if (y >= HALO && y < g.height - HALO && x >= HALO && x < g.width - HALO) {
                float m[5];
                blur_moments_v(c_win, s_h, ly, lx, m);
                // derivatives with b's blurred moments (mu_b, E[b^2], E[ab])
                const SsimTerms t = ssim_terms<1>(m, __ldg(head + H_C1), __ldg(head + H_C2));
                acc[1] = t.ssim;
                acc[2] = t.d_c1;
                acc[3] = t.d_c2;
                d_mu = t.d_mu;
                d_bb = t.d_xx;
                d_ab = t.d_ab;
            }
            const int64_t p = int64_t(y) * g.width + x, plane = int64_t(g.height) * g.width;
            maps[p] = d_mu;
            maps[plane + p] = d_bb;
            maps[2 * plane + p] = d_ab;
        }
    } else if (inside) {
        const int64_t p = int64_t(y) * g.width + x;
        const float d = kept(mask, g, y, x) ? norm_pred(__ldg(pred + p), g.norm, sub, div) - norm_gt(__ldg(gt + p), g.norm, div) : 0.f;
        acc[0] = g.l2 ? d * d : fabsf(d);
    }
    cta_sum_row(acc, s_red, threadIdx.x, [&] { return partials + (int64_t(blockIdx.y) * gridDim.x + blockIdx.x) * PART; });
}

__global__ void __launch_bounds__(RED_THREADS) depth_loss_kernel(DArgs g, int ssim, int64_t n_blocks, const float* __restrict__ partials,
                                                                 float* __restrict__ head, float* __restrict__ loss, float* __restrict__ stats) {
    __shared__ double s[RED_THREADS / 32][6];
    const int t = threadIdx.x, warp = t >> 5;
    const int nv = ssim ? 6 : 1;
    double v[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int64_t b = t; b < n_blocks; b += RED_THREADS)
        for (int k = 0; k < nv; ++k) v[k] += double(partials[b * PART + k]);
#pragma unroll
    for (int k = 0; k < 6; ++k) v[k] = warp_reduce<Sum>(v[k]);
    if ((t & 31) == 0) {
#pragma unroll
        for (int k = 0; k < 6; ++k) s[warp][k] = v[k];
    }
    __syncthreads();
    if (t != 0) return;
    for (int w = 1; w < RED_THREADS / 32; ++w)
        for (int k = 0; k < 6; ++k) v[k] += s[w][k];
    const double n = double(g.height) * g.width;
    const float lmean = float(v[0] / n);
    stats[0] = lmean;
    if (!ssim) {
        loss[0] = lmean;
        stats[1] = __int_as_float(0x7fffffff);          // no SSIM term: NaN
        head[H_VL] = float((g.l2 ? 2.0 : 1.0) / n);
        head[H_VS] = head[H_GMAX] = head[H_GMIN] = 0.f;
        return;
    }
    const double ns = double(g.height - 2 * HALO) * (g.width - 2 * HALO);
    const float smean = float(v[1] / ns);
    stats[1] = smean;
    loss[0] = (1.f - g.w) * lmean + g.w * (1.f - smean);
    // d loss / d dr = -w / ns * (sum dssim/dC1 * 2 k1^2 dr + sum dssim/dC2 * 2 k2^2 dr), shared by b's range
    const double dr = head[H_DR];
    const double kdr = -double(g.w) / ns * (v[2] * 2.0 * 1e-4 * dr + v[3] * 2.0 * 9e-4 * dr) * head[H_SHARE];
    head[H_GMAX] = float(kdr / v[4]);
    head[H_GMIN] = float(-kdr / v[5]);
    head[H_VL] = float((1.0 - g.w) / n);
    head[H_VS] = float(-double(g.w) / ns);
}

template <bool SSIM>
__global__ void __launch_bounds__(LT * LT) depth_bwd_kernel(DArgs g, const float* __restrict__ pred, const float* __restrict__ gt,
                                                            const uint8_t* __restrict__ mask, const float* __restrict__ head,
                                                            const float* __restrict__ maps, const float* __restrict__ v_loss,
                                                            float* __restrict__ v_pred) {
    __shared__ float s_m[SSIM ? 3 : 1][LE][LE];
    __shared__ float s_h[SSIM ? 3 : 1][LE][LT];
    const int x0 = blockIdx.x * LT, y0 = blockIdx.y * LT;
    const int lx = threadIdx.x % LT, ly = threadIdx.x / LT;
    const int x = x0 + lx, y = y0 + ly;
    float gm[3] = {0.f, 0.f, 0.f};
    if constexpr (SSIM) {
        const int64_t plane = int64_t(g.height) * g.width;
        load_halo(g.width, g.height, x0, y0, {s_m[0], s_m[1], s_m[2]}, [=](int m, int64_t p) { return __ldg(maps + m * plane + p); });
        __syncthreads();
        blur_maps_h(c_win, s_m, s_h);
        __syncthreads();
        blur_maps_v(c_win, s_h, ly, lx, gm);
    }
    if (x >= g.width || y >= g.height) return;
    const int64_t p = int64_t(y) * g.width + x;
    const float up = v_loss ? __ldg(v_loss) : 1.f;
    if (!kept(mask, g, y, x)) {
        v_pred[p] = 0.f;
        return;
    }
    const float sub = __ldg(head + H_SUB), div = __ldg(head + H_DIV);
    const float a = norm_gt(__ldg(gt + p), g.norm, div), b = norm_pred(__ldg(pred + p), g.norm, sub, div);
    const float d = b - a;
    const float sgn = d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f);          // torch.abs' subgradient at 0 is 0
    float v = __ldg(head + H_VL) * (g.l2 ? d : sgn);
    if (SSIM) {
        v += __ldg(head + H_VS) * ssim_grad(gm, b, a);
        if (b == __ldg(head + H_BMAX)) v += __ldg(head + H_GMAX);
        if (b == __ldg(head + H_BMIN)) v += __ldg(head + H_GMIN);
    }
    // chain through the normalisation: d pred' / d pred
    if (g.norm == 1 || g.norm == 3) v = __fdiv_rn(v, div);
    else if (g.norm == 2) v = v * div;
    v_pred[p] = up * v;
}

DArgs make_args(int height, int width, const uint8_t* mask, int64_t msy, int64_t msx, int loss_type, int norm, float median, float w) {
    DArgs g;
    g.height = height; g.width = width; g.l2 = loss_type == 1; g.norm = norm;
    g.msy = mask ? msy : 0; g.msx = mask ? msx : 0;
    g.median = median; g.w = w;
    return g;
}

int stat_blocks(int64_t n) { return int(div_up64(n, STAT_PIXELS) < STAT_MAX_BLOCKS ? div_up64(n, STAT_PIXELS) : STAT_MAX_BLOCKS); }
int64_t tile_blocks(int height, int width) { return int64_t(div_up(width, LT)) * div_up(height, LT); }

// the grid is (ceil(W/LT), ceil(H/LT)): ceil(H/LT) is at most 65535
bool depth_size_ok(int32_t height, int32_t width) {
    return height >= 1 && width >= 1 && height <= 65535 * LT && int64_t(height) * width <= INT32_MAX;
}

size_t depth_loss_workspace_bytes(int height, int width, int loss_type) {
    const int64_t n = int64_t(height) * width;
    int64_t floats = HEAD + int64_t(stat_blocks(n)) * STAT + tile_blocks(height, width) * PART;
    if (loss_type == 2) floats += 3 * n;
    return size_t(floats) * sizeof(float);
}

// pred, gt [H,W] contiguous; mask NULL or uint8 read at mask[msy y + msx x]; loss_type 0 l1, 1 l2, 2 l1+ssim; norm 0 none, 1 min-max,
// 2 median, 3 mean of gt.  The backward reads the workspace the forward wrote.  Shared by the forward and the backward; returns the
// error code, or 0 when the arguments are valid
int check_depth_loss(const char* fn, int32_t height, int32_t width, const float* pred, const float* gt, const uint8_t* mask, int64_t msy,
                     int64_t msx, int32_t loss_type, int32_t norm, const void* workspace, size_t workspace_bytes) {
    if (height < 1 || width < 1) return fail(fn, "image size must be >= 1");
    if (!depth_size_ok(height, width)) return fail(fn, "image too large");
    if (loss_type < 0 || loss_type > 2) return fail(fn, "loss_type must be 0 (l1), 1 (l2) or 2 (l1+ssim)");
    if (norm < 0 || norm > 3) return fail(fn, "norm must be 0 (none), 1 (min-max), 2 (median) or 3 (mean)");
    if (loss_type == 2 && (height < 11 || width < 11)) return fail(fn, "l1+ssim needs an image of at least 11x11");
    if (loss_type == 2 && mask) return fail(fn, "l1+ssim takes no mask");
    if (mask && (msy < 0 || msx < 0)) return fail(fn, "negative mask stride");
    if (!(pred && gt && workspace)) return fail(fn, "NULL pointer");
    if (workspace_bytes < depth_loss_workspace_bytes(height, width, loss_type)) return workspace_too_small(fn);
    return 0;
}

}  // namespace

}  // namespace b200gs

using namespace b200gs;

extern "C" {

size_t b200gs_depth_loss_workspace_bytes(int32_t height, int32_t width, int32_t loss_type) {
    if (!depth_size_ok(height, width) || loss_type < 0 || loss_type > 2) return 0;
    return depth_loss_workspace_bytes(height, width, loss_type);
}

int b200gs_depth_loss_fwd(int32_t height, int32_t width, const float* pred, const float* gt, const uint8_t* mask, int64_t msy, int64_t msx,
                          int32_t loss_type, int32_t norm, float median, float w, void* workspace, size_t workspace_bytes, float* loss,
                          float* stats, void* stream) {
    if (int rc = check_depth_loss(__func__, height, width, pred, gt, mask, msy, msx, loss_type, norm, workspace, workspace_bytes)) return rc;
    B200GS_CHECK_ARG(loss && stats, "NULL pointer");
    const cudaStream_t st = (cudaStream_t)stream;
    float* ws = static_cast<float*>(workspace);
    const DArgs g = make_args(height, width, mask, msy, msx, loss_type, norm, median, w);
    const int64_t n = int64_t(height) * width;
    // l1 and l2 without min-max or mean normalisation use no statistic: one CTA writes an empty partial
    const bool stats_needed = loss_type == 2 || norm == 1 || norm == 3;
    const int sb = stats_needed ? stat_blocks(n) : 1;
    float* stat_part = ws + HEAD;
    float* tile_part = stat_part + int64_t(stat_blocks(n)) * STAT;
    float* maps = tile_part + tile_blocks(height, width) * PART;
    depth_stats_kernel<<<sb, STAT_THREADS, 0, st>>>(stats_needed ? n : 0, pred, gt, stat_part);
    B200GS_LAUNCH_CHECK();
    depth_prep_kernel<<<1, RED_THREADS, 0, st>>>(g, sb, stat_part, ws);
    B200GS_LAUNCH_CHECK();
    const dim3 grid(div_up(width, LT), div_up(height, LT));
    if (loss_type == 2) depth_fwd_kernel<true><<<grid, LT * LT, 0, st>>>(g, pred, gt, mask, ws, maps, tile_part);
    else depth_fwd_kernel<false><<<grid, LT * LT, 0, st>>>(g, pred, gt, mask, ws, maps, tile_part);
    B200GS_LAUNCH_CHECK();
    depth_loss_kernel<<<1, RED_THREADS, 0, st>>>(g, loss_type == 2, tile_blocks(height, width), tile_part, ws, loss, stats);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

int b200gs_depth_loss_bwd(int32_t height, int32_t width, const float* pred, const float* gt, const uint8_t* mask, int64_t msy, int64_t msx,
                          int32_t loss_type, int32_t norm, float median, float w, const void* workspace, size_t workspace_bytes,
                          const float* v_loss, float* v_pred, void* stream) {
    if (int rc = check_depth_loss(__func__, height, width, pred, gt, mask, msy, msx, loss_type, norm, workspace, workspace_bytes)) return rc;
    B200GS_CHECK_ARG(v_pred, "NULL pointer");
    const float* ws = static_cast<const float*>(workspace);
    const DArgs g = make_args(height, width, mask, msy, msx, loss_type, norm, median, w);
    const int64_t n = int64_t(height) * width;
    const float* maps = ws + HEAD + int64_t(stat_blocks(n)) * STAT + tile_blocks(height, width) * PART;
    const dim3 grid(div_up(width, LT), div_up(height, LT));
    if (loss_type == 2) depth_bwd_kernel<true><<<grid, LT * LT, 0, (cudaStream_t)stream>>>(g, pred, gt, mask, ws, maps, v_loss, v_pred);
    else depth_bwd_kernel<false><<<grid, LT * LT, 0, (cudaStream_t)stream>>>(g, pred, gt, mask, ws, maps, v_loss, v_pred);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

}  // extern "C"
