// Warp-level 3xTF32 GEMM helpers shared by the MLP kernels (appearance.cu K20/K21, gs4d.cu K51): mma.sync.m16n8k8 TF32 with FP32
// accumulation, both operands split into a TF32 high part and the TF32 rounding of the remainder.
#pragma once

#include <cstdint>

namespace b200gs {

__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hi) : "f"(x));
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(lo) : "f"(x - __uint_as_float(hi)));
}

__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// c += a b with a = ah + al, b = bh + bl: the low-order products first
__device__ __forceinline__ void mma_3xtf32(float (&c)[4], const uint32_t (&ah)[4], const uint32_t (&al)[4], float b0, float b1) {
    uint32_t bh0, bl0, bh1, bl1;
    split_tf32(b0, bh0, bl0);
    split_tf32(b1, bh1, bl1);
    mma_tf32(c, al, bh0, bh1);
    mma_tf32(c, ah, bl0, bl1);
    mma_tf32(c, ah, bh0, bh1);
}

// One warp: acc[j] += A[16 x K] B[K x 8] for the n-tiles j < nt starting at column n0.  A is this warp's activation slice (row
// stride sa); B[k][n] = W[n sw + k] (the layer applied forward) or, TRANS, W[k sw + n] (its transpose: gradients to its input).
template <bool TRANS, int NT>
__device__ __forceinline__ void warp_gemm(const float* A, int sa, int K, const float* W, int sw, int n0, int nt, float (&acc)[NT][4], int lane) {
    const int g = lane >> 2, t = lane & 3;
    for (int k0 = 0; k0 < K; k0 += 8) {
        uint32_t ah[4], al[4];
        split_tf32(A[g * sa + k0 + t], ah[0], al[0]);
        split_tf32(A[(g + 8) * sa + k0 + t], ah[1], al[1]);
        split_tf32(A[g * sa + k0 + t + 4], ah[2], al[2]);
        split_tf32(A[(g + 8) * sa + k0 + t + 4], ah[3], al[3]);
#pragma unroll
        for (int j = 0; j < NT; ++j) {
            if (j < nt) {
                const int n = n0 + 8 * j + g;
                const float b0 = TRANS ? W[(k0 + t) * sw + n] : W[n * sw + k0 + t];
                const float b1 = TRANS ? W[(k0 + t + 4) * sw + n] : W[n * sw + k0 + t + 4];
                mma_3xtf32(acc[j], ah, al, b0, b1);
            }
        }
    }
}

template <int NT>
__device__ __forceinline__ void zero_acc(float (&acc)[NT][4]) {
#pragma unroll
    for (int j = 0; j < NT; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
}

}  // namespace b200gs
