// Shared device/host helpers for libb200gs (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/b200gs.h"

namespace b200gs {

void set_error(const char* fmt, ...);
void count_launch();   // every kernel launch of the library is counted (b200gs_launch_count): B200GS_LAUNCH_CHECK follows each <<<>>>

#define B200GS_CHECK_ARG(cond, msg)                                  \
    do {                                                              \
        if (!(cond)) {                                                \
            b200gs::set_error("%s: %s", __func__, msg);              \
            return B200GS_EINVAL;                                     \
        }                                                             \
    } while (0)

// set_error("<fn>: <msg>") and return rc.  For the check functions that several entry points share: with fn the entry point's
// __func__, the message reads as B200GS_CHECK_ARG's would
inline int fail(const char* fn, const char* msg, int rc = B200GS_EINVAL) {
    set_error("%s: %s", fn, msg);
    return rc;
}
inline int workspace_too_small(const char* fn) { return fail(fn, "workspace too small", B200GS_ENOSPACE); }

#define B200GS_CUDA(call)                                                                     \
    do {                                                                                       \
        cudaError_t _e = (call);                                                               \
        if (_e != cudaSuccess) {                                                               \
            b200gs::set_error("%s: %s failed: %s", __func__, #call, cudaGetErrorString(_e));  \
            return B200GS_ECUDA;                                                               \
        }                                                                                      \
    } while (0)

#define B200GS_LAUNCH_CHECK()                                                                  \
    do {                                                                                       \
        b200gs::count_launch();                                                                \
        cudaError_t _e = cudaGetLastError();                                                   \
        if (_e != cudaSuccess) {                                                               \
            b200gs::set_error("%s: kernel launch failed: %s", __func__, cudaGetErrorString(_e)); \
            return B200GS_ECUDA;                                                               \
        }                                                                                      \
    } while (0)

constexpr int TILE = B200GS_TILE;

__host__ __device__ inline int div_up(int a, int b) { return (a + b - 1) / b; }
inline int64_t div_up64(int64_t a, int64_t b) { return (a + b - 1) / b; }
inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// Tile rectangle touched by a splat: the two rules of SURVEY §8c.
//   vanilla (dgr getRect):   min = clamp(int((p - r)/16)),  max = clamp(int((p + r + 15)/16))
//   gsplat  (gaussian_projection.py:118-123): min = clamp(int((p - r)/16)),  max = clamp(int((p + r)/16) + 1)
// (int) truncates toward zero exactly like torch's .int(); clamp to [0, grid].
template <bool GSPLAT>
__device__ __forceinline__ void tile_rect(float x, float y, float r, int grid_x, int grid_y, int& x0, int& y0, int& x1, int& y1) {
    const float inv = 1.0f / float(TILE);  // exact power of two: same result as dividing
    x0 = min(grid_x, max(0, (int)((x - r) * inv)));
    y0 = min(grid_y, max(0, (int)((y - r) * inv)));
    if (GSPLAT) {
        x1 = min(grid_x, max(0, (int)((x + r) * inv) + 1));
        y1 = min(grid_y, max(0, (int)((y + r) * inv) + 1));
    } else {
        x1 = min(grid_x, max(0, (int)((x + r + float(TILE - 1)) * inv)));
        y1 = min(grid_y, max(0, (int)((y + r + float(TILE - 1)) * inv)));
    }
}

struct Sum { template <class T> __device__ __forceinline__ T operator()(T a, T b) const { return a + b; } };
struct Min { template <class T> __device__ __forceinline__ T operator()(T a, T b) const { return fmin(a, b); } };
struct Max { template <class T> __device__ __forceinline__ T operator()(T a, T b) const { return fmax(a, b); } };

// Reduction over the 32 lanes of a full warp by the xor butterfly 16, 8, 4, 2, 1: every lane gets the result, combined in the
// same order on every call.
template <class Op, class T>
__device__ __forceinline__ T warp_reduce(T v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = Op()(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

__device__ __forceinline__ float warp_sum(float v) { return warp_reduce<Sum>(v); }

// One row of K per-CTA partial sums from K values per thread (tid = the thread's index in the CTA of W full warps, of the caller's
// integer type): each value is summed over its warp, the warp sums go to s_red[warp][k], and thread k < K adds column k over
// warps 0, 1, ..., W - 1 in that order and stores it at row()[k], row() giving the CTA's output row.  Every thread of the CTA must
// call it (it synchronises the CTA); v is overwritten.
template <int W, int K, class Index, class Row>
__device__ __forceinline__ void cta_sum_row(float (&v)[K], float (&s_red)[W][K], Index tid, Row row) {
#pragma unroll
    for (int k = 0; k < K; ++k) v[k] = warp_sum(v[k]);
    if ((tid & 31) == 0) {
#pragma unroll
        for (int k = 0; k < K; ++k) s_red[tid >> 5][k] = v[k];
    }
    __syncthreads();
    if (tid < K) {
        float t = 0.f;
#pragma unroll
        for (int w = 0; w < W; ++w) t += s_red[w][tid];
        row()[tid] = t;
    }
}

// Stable LSD sort of uint2 {key, payload} records by the low `bits` bits of the key (knn.cu: a histogram launch, then one onesweep
// pass per 8 bits), a and b ping-pong buffers of n records; *out is the one that holds the result.  The scratch must be zero.
int record_key_bits(int64_t max_key);
size_t record_sort_scratch_bytes(int64_t n);
int launch_record_sort(int64_t n, int bits, uint2* a, uint2* b, void* scratch, cudaStream_t s, const uint2** out);

}  // namespace b200gs
