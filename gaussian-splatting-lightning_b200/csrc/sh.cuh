// Spherical-harmonic device code shared by every kernel that evaluates SH on a view direction: K1 / K8 and K15 (project.cu) and
// the Glossy-Gaussian colour-and-opacity kernels K47 / K48 (glossy.cu).  One copy of the constants, the basis polynomials of
// internal/utils/sh_utils.py:57-112, their derivatives, the coefficient loaders and the staged gradient-row stores.
#pragma once
#include "common.cuh"
#include "geometry.cuh"

namespace b200gs {

namespace {

constexpr float SH_C0 = 0.28209479177387814f;
constexpr float SH_C1 = 0.4886025119029199f;
__device__ constexpr float SH_C2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f,
                                       -1.0925484305920792f, 0.5462742152960396f};
__device__ constexpr float SH_C3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f, 0.3731763325901154f,
                                       -0.4570457994644658f, 1.445305721320277f, -0.5900435899266435f};
__device__ constexpr float SH_C4[9] = {2.5033429417967046f, -1.7701307697799304f, 0.9461746957575601f, -0.6690465435572892f,
                                       0.10578554691520431f, -0.6690465435572892f, 0.47308734787878004f, -1.7701307697799304f,
                                       0.6258357354491761f};

// Every kernel that touches SH coefficients is instantiated for MC = 16 (degrees 0..3, the common case: 48 coefficient
// registers) and MC = 25 (degree 4, sh_utils.py:102-111: 75 registers); each launcher picks the instantiation in one place.

// Loads the first ncoef*3 floats of one Gaussian's SH block into registers. 128-bit path when the block is 16B aligned.
template <int MC>
__device__ __forceinline__ void load_sh(const float* __restrict__ base, int ncoef, bool vec4, float* sh) {
    const int nf = ncoef * 3;
    if (vec4) {
        const float4* b4 = reinterpret_cast<const float4*>(base);
#pragma unroll
        for (int q = 0; q < MC * 3 / 4; ++q) {
            if (q * 4 < nf) {
                float4 t = __ldg(b4 + q);
                sh[q * 4 + 0] = t.x; sh[q * 4 + 1] = t.y; sh[q * 4 + 2] = t.z; sh[q * 4 + 3] = t.w;
            }
        }
    } else {
#pragma unroll
        for (int q = 0; q < MC * 3; ++q)
            if (q < nf) sh[q] = __ldg(base + q);
    }
}

// basis values for unit direction (x,y,z); writes (deg+1)^2 entries (sh_utils.py:57-112)
template <int MC>
__device__ __forceinline__ void sh_basis(int deg, float x, float y, float z, float* b) {
    b[0] = SH_C0;
    if (deg > 0) {
        b[1] = xm(-SH_C1, y); b[2] = xm(SH_C1, z); b[3] = xm(-SH_C1, x);
        if (deg > 1) {
            const float xx = xm(x, x), yy = xm(y, y), zz = xm(z, z), xy = xm(x, y), yz = xm(y, z), xz = xm(x, z);
            const float xx_yy = xa(xx, -yy);
            b[4] = xm(SH_C2[0], xy); b[5] = xm(SH_C2[1], yz); b[6] = xm(SH_C2[2], xa(xf(2.0f, zz, -xx), -yy));
            b[7] = xm(SH_C2[3], xz); b[8] = xm(SH_C2[4], xx_yy);
            if (deg > 2) {
                const float t4 = xa(xf(4.0f, zz, -xx), -yy);          // 4 zz - xx - yy
                b[9] = xm(xm(SH_C3[0], y), xf(3.0f, xx, -yy)); b[10] = xm(xm(SH_C3[1], xy), z);
                b[11] = xm(xm(SH_C3[2], y), t4); b[12] = xm(xm(SH_C3[3], z), xf(-3.0f, yy, xf(-3.0f, xx, xm(2.0f, zz))));
                b[13] = xm(xm(SH_C3[4], x), t4); b[14] = xm(xm(SH_C3[5], z), xx_yy);
                b[15] = xm(xm(SH_C3[6], x), xf(-3.0f, yy, xx));
                if (MC > 16 && deg > 3) {
                    const float s7 = xf(7.0f, zz, -1.0f), t7 = xf(7.0f, zz, -3.0f);
                    b[16] = xm(xm(SH_C4[0], xy), xx_yy); b[17] = xm(xm(SH_C4[1], yz), xf(3.0f, xx, -yy));
                    b[18] = xm(xm(SH_C4[2], xy), s7); b[19] = xm(xm(SH_C4[3], yz), t7);
                    b[20] = xm(SH_C4[4], xf(zz, xf(35.0f, zz, -30.0f), 3.0f)); b[21] = xm(xm(SH_C4[5], xz), t7);
                    b[22] = xm(xm(SH_C4[6], xx_yy), s7); b[23] = xm(xm(SH_C4[7], xz), xf(-3.0f, yy, xx));
                    b[24] = xm(SH_C4[8], xf(xx, xf(-3.0f, yy, xx), -xm(yy, xf(3.0f, xx, -yy))));
                }
            }
        }
    }
}

// d(basis)/d(x,y,z)
template <int MC>
__device__ __forceinline__ void sh_basis_grad(int deg, float x, float y, float z, float* bx, float* by, float* bz) {
    bx[0] = by[0] = bz[0] = 0.f;
    if (deg > 0) {
        bx[1] = 0.f; by[1] = -SH_C1; bz[1] = 0.f;
        bx[2] = 0.f; by[2] = 0.f; bz[2] = SH_C1;
        bx[3] = -SH_C1; by[3] = 0.f; bz[3] = 0.f;
        if (deg > 1) {
            bx[4] = SH_C2[0] * y; by[4] = SH_C2[0] * x; bz[4] = 0.f;
            bx[5] = 0.f; by[5] = SH_C2[1] * z; bz[5] = SH_C2[1] * y;
            bx[6] = SH_C2[2] * -2.f * x; by[6] = SH_C2[2] * -2.f * y; bz[6] = SH_C2[2] * 4.f * z;
            bx[7] = SH_C2[3] * z; by[7] = 0.f; bz[7] = SH_C2[3] * x;
            bx[8] = SH_C2[4] * 2.f * x; by[8] = SH_C2[4] * -2.f * y; bz[8] = 0.f;
            if (deg > 2) {
                const float xx = x * x, yy = y * y, zz = z * z;
                bx[9] = SH_C3[0] * 6.f * x * y; by[9] = SH_C3[0] * (3.f * xx - 3.f * yy); bz[9] = 0.f;
                bx[10] = SH_C3[1] * y * z; by[10] = SH_C3[1] * x * z; bz[10] = SH_C3[1] * x * y;
                bx[11] = SH_C3[2] * -2.f * x * y; by[11] = SH_C3[2] * (4.f * zz - xx - 3.f * yy); bz[11] = SH_C3[2] * 8.f * y * z;
                bx[12] = SH_C3[3] * -6.f * x * z; by[12] = SH_C3[3] * -6.f * y * z; bz[12] = SH_C3[3] * (6.f * zz - 3.f * xx - 3.f * yy);
                bx[13] = SH_C3[4] * (4.f * zz - 3.f * xx - yy); by[13] = SH_C3[4] * -2.f * x * y; bz[13] = SH_C3[4] * 8.f * x * z;
                bx[14] = SH_C3[5] * 2.f * x * z; by[14] = SH_C3[5] * -2.f * y * z; bz[14] = SH_C3[5] * (xx - yy);
                bx[15] = SH_C3[6] * (3.f * xx - 3.f * yy); by[15] = SH_C3[6] * -6.f * x * y; bz[15] = 0.f;
                if (MC > 16 && deg > 3) {
                    const float xyz = x * y * z, s7 = 7.f * zz - 1.f, t7 = 7.f * zz - 3.f, u21 = 21.f * zz - 3.f;
                    bx[16] = SH_C4[0] * y * (3.f * xx - yy); by[16] = SH_C4[0] * x * (xx - 3.f * yy); bz[16] = 0.f;
                    bx[17] = SH_C4[1] * 6.f * xyz; by[17] = SH_C4[1] * 3.f * z * (xx - yy); bz[17] = SH_C4[1] * y * (3.f * xx - yy);
                    bx[18] = SH_C4[2] * y * s7; by[18] = SH_C4[2] * x * s7; bz[18] = SH_C4[2] * 14.f * xyz;
                    bx[19] = 0.f; by[19] = SH_C4[3] * z * t7; bz[19] = SH_C4[3] * y * u21;
                    bx[20] = 0.f; by[20] = 0.f; bz[20] = SH_C4[4] * z * (140.f * zz - 60.f);
                    bx[21] = SH_C4[5] * z * t7; by[21] = 0.f; bz[21] = SH_C4[5] * x * u21;
                    bx[22] = SH_C4[6] * 2.f * x * s7; by[22] = SH_C4[6] * -2.f * y * s7; bz[22] = SH_C4[6] * 14.f * z * (xx - yy);
                    bx[23] = SH_C4[7] * 3.f * z * (xx - yy); by[23] = SH_C4[7] * -6.f * xyz; bz[23] = SH_C4[7] * x * (xx - 3.f * yy);
                    bx[24] = SH_C4[8] * 4.f * x * (xx - 3.f * yy); by[24] = SH_C4[8] * 4.f * y * (yy - 3.f * xx); bz[24] = 0.f;
                }
            }
        }
    }
}

// (dx, dy, dz) /= max(|(dx, dy, dz)|, 1e-12), F.normalize's floor (gsplat normalises the same way); returns the factor.  A zero
// vector stays the zero direction.
__device__ __forceinline__ float normalize_dir(float& dx, float& dy, float& dz) {
    const float inv_len = 1.0f / fmaxf(sqrtf(dx * dx + dy * dy + dz * dz), 1e-12f);
    dx *= inv_len; dy *= inv_len; dz *= inv_len;
    return inv_len;
}

// SH block of Gaussian i into registers: [K,3] contiguous, or dc [1,3] + rest [K-1,3] when RAW
template <bool RAW, int MC>
__device__ __forceinline__ void load_sh_any(const float* __restrict__ shs, const float* __restrict__ shs_rest, int64_t i, int stride,
                                            int ncoef, float* sh) {
    if (RAW) {
        sh[0] = __ldg(shs + 3 * i); sh[1] = __ldg(shs + 3 * i + 1); sh[2] = __ldg(shs + 3 * i + 2);
        const float* r = shs_rest + i * int64_t(stride - 1) * 3;
#pragma unroll
        for (int q = 3; q < MC * 3; ++q)
            if (q < ncoef * 3) sh[q] = __ldg(r + q - 3);
    } else {
        load_sh<MC>(shs + i * int64_t(stride) * 3, ncoef, ((stride * 3) & 3) == 0, sh);
    }
}

// Gradient of the SH colour with respect to the point the unit view direction (dx, dy, dz) = (p - campos) * inv_len starts from, given
// the weights w[k] = <SH coefficient k, dL/drgb> for k >= 1: sum_k w[k] d(basis_k)/d(dir), less its radial component, times inv_len.
template <int MC>
__device__ __forceinline__ float3 view_dir_grad(int deg, float dx, float dy, float dz, float inv_len, const float* w) {
    const int ncoef = (deg + 1) * (deg + 1);
    float bx[MC], by[MC], bz[MC];
    sh_basis_grad<MC>(deg, dx, dy, dz, bx, by, bz);
    float ddx = 0.f, ddy = 0.f, ddz = 0.f;
#pragma unroll
    for (int k = 1; k < MC; ++k) {
        if (k < ncoef) { ddx += bx[k] * w[k]; ddy += by[k] * w[k]; ddz += bz[k] * w[k]; }
    }
    const float dot = dx * ddx + dy * ddy + dz * ddz;
    return make_float3((ddx - dx * dot) * inv_len, (ddy - dy * dot) * inv_len, (ddz - dz * dot) * inv_len);
}

// SH-gradient rows of a warp's 32 Gaussians, staged in shared memory (row of lane l at s_rows_warp + l * (rw | 1); the odd stride
// keeps the staging conflict-free), written back with fully coalesced 128-bit stores.  Every row is written (zeros for culled
// Gaussians), so the warp's rows are one contiguous span of the output (5.6-6 KB at 45-48 floats per row).  ACC: added to dst_base.
__device__ __forceinline__ void flush_sh_rows(const float* s_rows_warp, int rw, int64_t i, int64_t n, unsigned lane, float* __restrict__ dst_base,
                                              bool ACC) {
    const int rwp = rw | 1;
    __syncwarp();
    const int64_t i0 = i - lane;
    const int rows_valid = (i0 < n) ? (int)min((int64_t)32, n - i0) : 0;
    const int total = rows_valid * rw;
    float* dst = dst_base + i0 * rw;
    const float* sw = s_rows_warp;
    if ((reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
        for (int idx = lane; idx * 4 + 3 < total; idx += 32) {
            int f = idx * 4, r = f / rw, c = f - r * rw;
            float t[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                t[e] = sw[r * rwp + c];
                if (++c == rw) { c = 0; ++r; }
            }
            if (ACC) {
                const float4 old = reinterpret_cast<const float4*>(dst)[idx];
                t[0] += old.x; t[1] += old.y; t[2] += old.z; t[3] += old.w;
            }
            reinterpret_cast<float4*>(dst)[idx] = make_float4(t[0], t[1], t[2], t[3]);
        }
        for (int f = (total & ~3) + lane; f < total; f += 32) dst[f] = sw[(f / rw) * rwp + f % rw] + (ACC ? dst[f] : 0.f);
    } else {
        for (int f = lane; f < total; f += 32) dst[f] = sw[(f / rw) * rwp + f % rw] + (ACC ? dst[f] : 0.f);
    }
}

}  // namespace

}  // namespace b200gs
