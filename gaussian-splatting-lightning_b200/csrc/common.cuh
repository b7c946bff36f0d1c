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

__device__ __forceinline__ float warp_sum(float v) {
    v += __shfl_xor_sync(0xffffffffu, v, 16);
    v += __shfl_xor_sync(0xffffffffu, v, 8);
    v += __shfl_xor_sync(0xffffffffu, v, 4);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v;
}

// launchers (one per translation unit)
int launch_project_fwd(const B200gsView& v, int64_t n, const float* means, const float* scales, const float* quats,
                       const float* shs, float* xy, float* depth, int32_t* radii, float* conic, float* comp,
                       int32_t* tiles, float* cov3d, float* rgb, uint8_t* clamped, cudaStream_t s);
int launch_project_bwd(const B200gsView& v, int64_t n, const float* means, const float* scales, const float* quats,
                       const float* shs, const int32_t* radii, const uint8_t* clamped, const float* v_xy,
                       const float* v_depth, const float* v_conic, const float* v_comp, const float* v_rgb,
                       float* v_means, float* v_scales, float* v_quats, float* v_shs, cudaStream_t s);
int launch_project_fwd_rows(const B200gsView& v, int64_t n, const float* means, const float* log_scales, const float* raw_quats,
                            const float* opac_logits, const float* shs_dc, const float* shs_rest, int anti_aliased, float* rows,
                            int32_t* radii, uint8_t* clamped, int32_t* tiles, cudaStream_t s);
int launch_project_bwd_rows(const B200gsView& v, int64_t n, const float* means, const float* log_scales, const float* raw_quats,
                            const float* opac_logits, const float* shs_dc, const float* shs_rest, int anti_aliased, const int32_t* radii,
                            const uint8_t* clamped, const int32_t* row_offsets, const float* v_rows, int accumulate, float* v_means,
                            float* v_log_scales, float* v_raw_quats, float* v_opac_logit, float* v_shs_dc, float* v_shs_rest,
                            float* v_mean2d, int v_mean2d_cols, cudaStream_t s);
int launch_project_fwd_multi(const B200gsView* views, int n_views, int64_t n, const float* means, const float* scales, const float* quats,
                             const float* opac_logits, const float* shs_dc, const float* shs_rest, int anti_aliased, float* xy, float* depth,
                             int32_t* radii, float* conic, float* rgb, uint8_t* clamped, float* opac_out, cudaStream_t s);
size_t project_pack_workspace_bytes(int n_views, int64_t n);
int launch_project_pack_multi(const B200gsView* views, int n_views, int64_t n, const float* means, const float* scales, const float* quats,
                              const float* opac_logits, const float* shs_dc, const float* shs_rest, int anti_aliased, float* xy, int32_t* radii,
                              uint8_t* clamped, int32_t* row_index, float* const* dst_rows, int64_t cap, void* workspace, size_t workspace_bytes,
                              int64_t* d_count, cudaStream_t s);
int launch_project_bwd_multi(const B200gsView* views, int n_views, int64_t n, const float* means, const float* scales, const float* quats,
                             const float* opac_logits, const float* shs_rest, int anti_aliased, const int32_t* radii, const uint8_t* clamped,
                             const int32_t* row_index, const float* const* v_rows, float* v_means, float* v_scales, float* v_quats,
                             float* v_opac_logit, float* v_shs_dc, float* v_shs_rest, cudaStream_t s);
// split = true: coeffs / v_coeffs are dc [n,1,3], rest / v_rest [n,stride-1,3] read and written in place, mask[n] (nullable) zeroes rows
int launch_sh_fwd(int degree, int stride, int64_t n, const float* dirs, const float* coeffs, float* rgb, cudaStream_t s, bool split = false,
                  const float* rest = nullptr, const uint8_t* mask = nullptr);
int launch_sh_bwd(int degree, int stride, int64_t n, const float* dirs, const float* coeffs, const float* v_rgb,
                  float* v_coeffs, float* v_dirs, cudaStream_t s, bool split = false, const float* rest = nullptr,
                  const uint8_t* mask = nullptr, float* v_rest = nullptr);
// gsplat isect_ids / isect_offset_encode for one camera (isect.cu)
int launch_isect_keys(int n_tiles, const int32_t* tile_ranges, const int32_t* sorted_ids, int64_t n_pairs, const float* depth, int64_t* keys,
                      cudaStream_t s);
int launch_isect_offsets(int64_t n_pairs, const int64_t* keys, int n_tiles, int32_t* offsets, cudaStream_t s);

size_t bin_count_workspace_bytes(int64_t n);
size_t bin_sort_workspace_bytes(int64_t n, int64_t max_coarse, int width, int height);
// rows: xy, depth, radii, conic and opacity are columns of one 16-byte aligned [n,12] row buffer (b200gs.h), optionally in
// blocks of block_rows rows of which the first block_counts[b] are valid; otherwise separate arrays, conic and opacity NULL
// without culling
int bin_count(int mode, int width, int height, int64_t n, bool rows, const float* xy, const float* depth, const int32_t* radii,
              const float* conic, const float* opacity, void* ws, size_t ws_bytes, int64_t* d_counts, int64_t* host_counts,
              int sync_host, cudaStream_t s, const int64_t* block_counts = nullptr, int64_t block_rows = 0);
int publish_i64(const int64_t* d_values, int64_t* host_values, int n, cudaStream_t s);
size_t pack_rows_workspace_bytes(int64_t n);
int pack_rows(int64_t n, const float* xy, const float* depth, const float* conic, const float* comp, const float* opacity,
              const float* rgb, const int32_t* radii, void* ws, int32_t* row_index, float* rows, int64_t* d_count, cudaStream_t s);
int bin_sort(int mode, int width, int height, int64_t n, int cull, int64_t max_coarse, int64_t max_pairs, int64_t* d_counts,
             const void* ws_a, void* ws_b, size_t ws_b_bytes, int32_t* sorted_ids, int32_t* tile_ranges, int64_t* host_counts,
             int sync_host, cudaStream_t s);

int launch_selective_adam(int64_t rows, int width, float* param, const float* grad, float* exp_avg, float* exp_avg_sq, const uint8_t* visible,
                          float lr, float b1, float b2, float eps, cudaStream_t s);
int launch_densify_stats(int64_t n, const int32_t* radii, const uint8_t* visible, const float* grad, int grad_stride, float sx, float sy,
                         float* max_radii2d, float* grad_accum, float* denom, cudaStream_t s);

int launch_mcmc_relocation(int64_t n, const float* opacities, const float* scales, const int32_t* counts, int n_max, float* new_opacities,
                           float* new_scales, cudaStream_t s);
int launch_mcmc_position_noise(int64_t n, float* means, const float* log_scales, const float* raw_quats, const float* opacity_logits,
                               float scale, uint64_t seed, uint64_t offset, cudaStream_t s);

// bilateral grid (bilagrid.cu): grids [n_grids,12,L,gh,gw]; xy [batch,height,width,2]; rgb / out / v_out / v_rgb share the element
// strides (sb, sy, sx, sc); grid_idx int64 [n_idx], n_idx == 1 (broadcast) or batch
int launch_bilagrid_slice_fwd(int n_grids, int L, int gh, int gw, const float* grids, int batch, int height, int width, const float* xy,
                              const float* rgb, int64_t sb, int64_t sy, int64_t sx, int64_t sc, const int64_t* grid_idx, int n_idx,
                              float* out, cudaStream_t s);
int launch_bilagrid_slice_bwd(int n_grids, int L, int gh, int gw, const float* grids, int batch, int height, int width, const float* xy,
                              const float* rgb, int64_t sb, int64_t sy, int64_t sx, int64_t sc, const int64_t* grid_idx, int n_idx,
                              const float* v_out, float* v_rgb, float* v_grids, cudaStream_t s);
int64_t bilagrid_tv_blocks(int n, int channels, int L, int gh, int gw);
int launch_bilagrid_tv_fwd(int n, int channels, int L, int gh, int gw, const float* grids, float* partials, cudaStream_t s);
int launch_bilagrid_tv_bwd(int n, int channels, int L, int gh, int gw, const float* grids, const float* v_tv, float* v_grids,
                           cudaStream_t s);

// exposure correction (exposure.cu): render / out / v_out / v_render [3,H,W] through the element strides (sc, sy, sx); params
// [n_app, n_params] (n_params 4 or 7: with bias); the id read from id_dev when not NULL, else id_host; shade [s, s] (s = 0: none)
size_t exposure_workspace_bytes(int height, int width, int shade_size, bool backward);
int launch_exposure_fwd(int height, int width, const float* render, int64_t sc, int64_t sy, int64_t sx, int n_app, int n_params,
                        const float* params, const int64_t* id_dev, int64_t id_host, int s, const float* shade, float max_gray,
                        float max_gamma, float* ws, float* out, cudaStream_t st);
int launch_exposure_bwd(int height, int width, const float* render, int64_t sc, int64_t sy, int64_t sx, int n_app, int n_params,
                        const float* params, const int64_t* id_dev, int64_t id_host, int s, const float* shade, float max_gray,
                        float max_gamma, float* ws, const float* v_out, float* v_render, float* v_params, float* v_shade,
                        cudaStream_t st);

// appearance MLP (appearance.cu); the shape arguments are those of B200gsAppearanceMlp, validated by the caller
bool appearance_mlp_fits(int feat_dim, int n_freq, int n_neurons, int n_layers, int n_out);
size_t appearance_mlp_workspace_bytes(int feat_dim, int n_freq, int n_neurons, int n_layers, int n_out);
int launch_appearance_mlp_fwd(const B200gsAppearanceMlp& m, int64_t n, const float* features, const uint8_t* mask, const float* base_rgb,
                              const float* dirs, const float* cam, const float* raw_opacity, float* out, float* opacity_offsets,
                              float* opacities, cudaStream_t s);
int launch_appearance_mlp_bwd(const B200gsAppearanceMlp& m, int64_t n, const float* features, const uint8_t* mask, const float* base_rgb,
                              const float* dirs, const float* cam, const float* raw_opacity, const float* v_out, const float* v_opacities,
                              const float* v_opacity_offsets, float* v_base_rgb, float* v_features, float* v_raw_opacity, float* workspace,
                              float* v_params, cudaStream_t s);

size_t knn_workspace_bytes(int64_t n);
int launch_knn_mean_dist2(int64_t n, const float* points, float* out, void* ws, size_t ws_bytes, cudaStream_t s);

int64_t loss_blocks(int channels, int width, int height);
int launch_loss_fwd(int channels, int width, int height, const float* img, const float* gt, float* dmaps, float* partials, cudaStream_t s);
int launch_loss_bwd(int channels, int width, int height, const float* img, const float* gt, const float* dmaps, float lambda_dssim,
                    const float* v_loss, float* v_img, cudaStream_t s);

// rows: xy, conic, opacity and colors (and the gradient outputs) are columns of 16-byte aligned [n,12] row buffers, channels == 3
int launch_blend_fwd(int mode, int width, int height, int channels, const int32_t* ranges, const int32_t* ids,
                     bool rows, const float* xy, const float* conic, const float* opacity, const float* colors, const float* bg,
                     float* image, int64_t pix_stride, int64_t ch_stride, float* final_T, int32_t* n_contrib,
                     float* alpha, cudaStream_t s, uint8_t* hit_any = nullptr);
int launch_blend_bwd(int mode, int width, int height, int channels, const int32_t* ranges, const int32_t* ids,
                     bool rows, const float* xy, const float* conic, const float* opacity, const float* colors, const float* bg,
                     const float* final_T, const int32_t* n_contrib, const float* v_image, int64_t pix_stride,
                     int64_t ch_stride, const float* v_alpha, float sx, float sy, float* v_xy, float* v_conic,
                     float* v_opacity, float* v_colors, float* v_xy_abs, cudaStream_t s);
// gsplat mode, any channel count >= 1 (chunks of 32); [n, channels] features, [H, W, channels] image; v_xy == NULL: features only
int launch_blend_feat_fwd(int width, int height, int channels, const int32_t* ranges, const int32_t* ids, const float* xy, const float* conic,
                          const float* opacity, const float* features, const float* bg, float* image, float* final_T, int32_t* n_contrib,
                          float* alpha, cudaStream_t s);
int launch_blend_feat_bwd(int width, int height, int channels, const int32_t* ranges, const int32_t* ids, const float* xy, const float* conic,
                          const float* opacity, const float* features, const float* bg, const float* final_T, const int32_t* n_contrib,
                          const float* v_image, const float* v_alpha, float* v_features, float* v_xy, float* v_conic, float* v_opacity,
                          float* v_xy_abs, cudaStream_t s);

}  // namespace b200gs
