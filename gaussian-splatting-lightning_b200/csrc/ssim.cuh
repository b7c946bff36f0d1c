// SSIM tile engine of the L1+SSIM training loss (loss.cu, K9/K10) and the inverse-depth loss (depth_loss.cu, K29/K31).
// One CTA of LT x LT threads per 16x16 tile holds the tile and its HALO-pixel border in shared memory, blurs with the separable
// TAPS-tap window horizontally over the border rows into s_h[map][LE][LT], then vertically at each pixel of the tile.  The
// window is the caller's __constant__ table: the two losses use windows that differ in their last bits (the reference's
// ssim.py and torchmetrics'), and each keeps its own.
#pragma once
#include "common.cuh"

namespace b200gs {

constexpr int LT = 16;             // tile edge
constexpr int HALO = 5;            // (TAPS - 1) / 2
constexpr int LE = LT + 2 * HALO;  // 26: tile edge with the halo
constexpr int TAPS = 11;

using Window = float[TAPS];

// The reference's internal/utils/ssim.py SSIM (the L1+SSIM training loss, K9/K10, and its visibility-masked form, K34/K35):
// C1 = 0.01^2, C2 = 0.03^2 and the 11-tap sigma-1.5 window in float32 exactly as the reference builds it (exp in double, cast to
// float32, divided by its float32 sum).  A __constant__ table per translation unit that includes this header.
constexpr float SSIM_C1 = 0.01f * 0.01f;
constexpr float SSIM_C2 = 0.03f * 0.03f;
namespace {
__device__ __constant__ float c_ssim_win[TAPS] = {1.028380124e-03f, 7.598758209e-03f, 3.600077331e-02f, 1.093606874e-01f, 2.130055279e-01f,
                                                  2.660117149e-01f, 2.130055279e-01f, 1.093606874e-01f, 3.600077331e-02f, 7.598758209e-03f,
                                                  1.028380124e-03f};
}  // namespace

// dst[m] = the (LE x LE) halo tile of the tile at (x0, y0): load(m, p) at the image's pixel p = y * width + x, 0 outside the image
template <int N, class Load>
__device__ __forceinline__ void load_halo(int width, int height, int x0, int y0, float (*const (&dst)[N])[LE], Load load) {
    for (int i = threadIdx.x; i < LE * LE; i += LT * LT) {
        const int ly = i / LE, lx = i - ly * LE;
        const int x = x0 + lx - HALO, y = y0 + ly - HALO;
        const bool in = x >= 0 && x < width && y >= 0 && y < height;
#pragma unroll
        for (int m = 0; m < N; ++m) dst[m][ly][lx] = in ? load(m, int64_t(y) * width + x) : 0.f;
    }
}

// horizontal pass of the five moments (a, b, a^2, b^2, ab) over the halo rows: h[5][LE][LT]
__device__ __forceinline__ void blur_moments_h(const Window& win, const float (*a)[LE], const float (*b)[LE], float (*h)[LE][LT]) {
    for (int i = threadIdx.x; i < LE * LT; i += LT * LT) {
        const int ly = i / LT, lx = i - ly * LT;
        float m0 = 0.f, m1 = 0.f, m2 = 0.f, m3 = 0.f, m4 = 0.f;
#pragma unroll
        for (int k = 0; k < TAPS; ++k) {
            const float w = win[k], va = a[ly][lx + k], vb = b[ly][lx + k];
            m0 = fmaf(w, va, m0);
            m1 = fmaf(w, vb, m1);
            m2 = fmaf(w, va * va, m2);
            m3 = fmaf(w, vb * vb, m3);
            m4 = fmaf(w, va * vb, m4);
        }
        h[0][ly][lx] = m0; h[1][ly][lx] = m1; h[2][ly][lx] = m2; h[3][ly][lx] = m3; h[4][ly][lx] = m4;
    }
}

// vertical pass at the tile's pixel (lx, ly) of the five moments: m = (mu_a, mu_b, E[a^2], E[b^2], E[ab])
__device__ __forceinline__ void blur_moments_v(const Window& win, const float (*h)[LE][LT], int ly, int lx, float (&m)[5]) {
    m[0] = m[1] = m[2] = m[3] = m[4] = 0.f;
#pragma unroll
    for (int k = 0; k < TAPS; ++k) {
        const float w = win[k];
        m[0] = fmaf(w, h[0][ly + k][lx], m[0]);
        m[1] = fmaf(w, h[1][ly + k][lx], m[1]);
        m[2] = fmaf(w, h[2][ly + k][lx], m[2]);
        m[3] = fmaf(w, h[3][ly + k][lx], m[3]);
        m[4] = fmaf(w, h[4][ly + k][lx], m[4]);
    }
}

// the backward's horizontal pass of the three derivative maps' halo tiles over the halo rows: h[3][LE][LT]
__device__ __forceinline__ void blur_maps_h(const Window& win, const float (*src)[LE][LE], float (*h)[LE][LT]) {
    for (int i = threadIdx.x; i < LE * LT; i += LT * LT) {
        const int ly = i / LT, lx = i - ly * LT;
        float h0 = 0.f, h1 = 0.f, h2 = 0.f;
#pragma unroll
        for (int k = 0; k < TAPS; ++k) {
            const float w = win[k];
            h0 = fmaf(w, src[0][ly][lx + k], h0);
            h1 = fmaf(w, src[1][ly][lx + k], h1);
            h2 = fmaf(w, src[2][ly][lx + k], h2);
        }
        h[0][ly][lx] = h0; h[1][ly][lx] = h1; h[2][ly][lx] = h2;
    }
}

// the backward's vertical pass at the tile's pixel (lx, ly): g = the window applied to the three derivative maps
__device__ __forceinline__ void blur_maps_v(const Window& win, const float (*h)[LE][LT], int ly, int lx, float (&g)[3]) {
    g[0] = g[1] = g[2] = 0.f;
#pragma unroll
    for (int k = 0; k < TAPS; ++k) {
        const float w = win[k];
        g[0] = fmaf(w, h[0][ly + k][lx], g[0]);
        g[1] = fmaf(w, h[1][ly + k][lx], g[1]);
        g[2] = fmaf(w, h[2][ly + k][lx], g[2]);
    }
}

struct SsimTerms {
    float ssim;
    float d_c1, d_c2;                  // d ssim / d C1, d C2
    float d_mu, d_xx, d_ab;            // d ssim / d (mu_x, E[x^2], E[ab])
};

// SSIM at one pixel from its blurred moments m = (mu_a, mu_b, E[a^2], E[b^2], E[ab]), and its derivatives with the constants and
// with the blurred moments of the operand x (X = 0: a, 1: b) as independent variables; the variances depend on mu_x through
// -mu_x^2 and -mu_a mu_b.  x is selected, not swapped in: the map's expressions keep their operand order, and with it the
// rounding of their contracted multiply-adds.
template <int X>
__device__ __forceinline__ SsimTerms ssim_terms(const float (&m)[5], float C1, float C2) {
    const float mu1 = m[0], mu2 = m[1], e11 = m[2], e22 = m[3], e12 = m[4];
    const float s1 = e11 - mu1 * mu1, s2 = e22 - mu2 * mu2, s12 = e12 - mu1 * mu2;
    const float A1 = 2.f * mu1 * mu2 + C1, A2 = 2.f * s12 + C2;
    const float B1 = mu1 * mu1 + mu2 * mu2 + C1, B2 = s1 + s2 + C2;
    const float iB1 = 1.f / B1, iB2 = 1.f / B2;
    const float mx = X == 0 ? mu1 : mu2, my = X == 0 ? mu2 : mu1;
    SsimTerms t;
    t.ssim = A1 * A2 * iB1 * iB2;
    t.d_c1 = A2 * iB1 * iB2 - t.ssim * iB1;
    t.d_c2 = A1 * iB1 * iB2 - t.ssim * iB2;
    t.d_mu = (2.f * my * A2 - 2.f * my * A1) * iB1 * iB2 - t.ssim * (2.f * mx * iB1 - 2.f * mx * iB2);
    t.d_xx = -t.ssim * iB2;
    t.d_ab = 2.f * A1 * iB1 * iB2;
    return t;
}

// d (sum of the SSIM map) / d x at a pixel, from g = the window applied to the three derivative maps (d_mu, d_xx, d_ab) (the
// window is symmetric); y is the other operand
__device__ __forceinline__ float ssim_grad(const float (&g)[3], float x, float y) { return g[0] + 2.f * x * g[1] + y * g[2]; }

}  // namespace b200gs
