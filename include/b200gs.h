/*
 * b200gs — C ABI of the sm_90a (H100) differentiable 3D-Gaussian rasterizer (libb200gs.so).
 *
 * This is the drop-in boundary for the hot path of yzslab/gaussian-splatting-lightning.  The reference has no
 * native code of its own: its renderers call two pip extensions through Python, and these entry points are what a
 * binding for those call sites needs (citations relative to the reference repository):
 *
 *   diff_gaussian_rasterization.GaussianRasterizer(...)(means3D, means2D, shs, colors_precomp, opacities, scales,
 *       rotations, cov3D_precomp) -> (color, radii)            internal/renderers/vanilla_renderer.py:62-77,111-120
 *   gsplat.v0_interfaces.project_gaussians(...) -> 7-tuple     internal/renderers/gsplat_renderer.py:64-79
 *   gsplat.sh.spherical_harmonics(deg, dirs, coeffs)           internal/renderers/gsplat_renderer.py:105
 *   gsplat.rasterize.rasterize_gaussians(...) -> [H,W,D](,alpha)  internal/renderers/gsplat_renderer.py:86-99
 *   gsplat.cuda._wrapper / gsplat.sh_decomposed / gsplat.cuda.isect_tiles_tile_based_culling / rasterize_to_pixels
 *                                                              internal/renderers/gsplat_v1_renderer.py:8-20
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless named host_*; all floating point is fp32, contiguous.
 *   - the library never allocates or frees device memory: the caller (PyTorch's caching allocator) owns every
 *     buffer including the workspace -> no hidden cudaMalloc, no hidden synchronisation (except where stated).
 *   - all work is enqueued on the cudaStream_t passed as `stream` (a CUstream handle; pass
 *     torch.cuda.current_stream().cuda_stream).
 *   - return 0 on success, a negative B200GS_E* code on failure; b200gs_last_error() gives a thread-local message.
 *     Nothing throws across the ABI; nothing calls exit().  Re-entrant: no global mutable state.
 *   - "mode": B200GS_MODE_VANILLA = diff-gaussian-rasterization semantics (near 0.2, mean2D via the NDC projection
 *     matrix, pixel sample at integer coords, alpha clamp 0.99 straight-through, stop T<1e-4, rect max uses +15);
 *     B200GS_MODE_GSPLAT = the semantics of internal/utils/gaussian_projection.py + gsplat's rasterizer (near 0.01,
 *     K t/(z+1e-6), blur compensation, pixel centres +0.5, alpha clamp 0.999 as a true clamp, stop T<=1e-4,
 *     rect max = int((p+r)/16)+1).
 */
#ifndef B200GS_H
#define B200GS_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define B200GS_API __attribute__((visibility("default")))
#else
#define B200GS_API
#endif

#define B200GS_MODE_VANILLA 0
#define B200GS_MODE_GSPLAT 1

#define B200GS_OK 0
#define B200GS_EINVAL (-1)    /* bad argument (null pointer, bad size, unsupported degree/channels) */
#define B200GS_ECUDA (-2)     /* a CUDA call or launch failed; message holds cudaGetErrorString */
#define B200GS_ENOSPACE (-3)  /* workspace or pair capacity too small */

#define B200GS_TILE 16

/* One view.  Matrices are stored exactly as the reference's Camera stores them (cameras.py:147-189):
 * viewmatrix = world_to_camera, "transposed" (row-major [4][4], translation in the last ROW; p_cam = p * M[:3,:3] + M[3,:3]);
 * projmatrix = full_projection = world_to_camera @ projection (same layout; vanilla mode only). */
typedef struct B200gsView {
    int32_t width;
    int32_t height;
    int32_t mode;           /* B200GS_MODE_* */
    int32_t sh_degree;      /* active degree 0..4 */
    int32_t sh_stride;      /* coefficients stored per Gaussian (K of shs[N,K,3]); >= (sh_degree+1)^2 */
    int32_t reserved0;
    float fx, fy, cx, cy;   /* gsplat mode intrinsics (gsplat_renderer.py:70-73) */
    float tanfovx, tanfovy; /* vanilla mode (vanilla_renderer.py:59-60) */
    float scale_modifier;
    float eps2d;            /* 2D low-pass added to the cov2D diagonal: 0.3 */
    float near_plane;       /* <=0 selects the mode default (0.2 vanilla / 0.01 gsplat) */
    float reserved1;
    float viewmatrix[16];
    float projmatrix[16];
    float campos[3];
    float reserved2;
} B200gsView;

B200GS_API const char* b200gs_last_error(void);
B200GS_API int b200gs_version(void);
/* number of CUDA kernels this library has launched in this process (monotonic; every launch site increments it) */
B200GS_API int64_t b200gs_launch_count(void);

/* ---- K1: per-Gaussian projection (+ optional fused SH colour) ------------------------------------------------
 * replaces dgr preprocessCUDA / gsplat project_gaussians (+ spherical_harmonics when shs != NULL).
 * in : means[n,3] scales[n,3] quats[n,4] (wxyz, used as given); shs[n,sh_stride,3] or NULL.
 * out: xy[n,2] depth[n] radii[n] conic[n,3] tiles[n]; comp[n] (gsplat, nullable); cov3d[n,6] upper triangle (nullable);
 *      rgb[n,3] = max(SH+0.5,0) and clamped[n] (bit c set when channel c was clamped) when shs != NULL.
 *      Culled Gaussians get zeros everywhere (radii 0, tiles 0).
 * SH view direction: normalize(mean - campos).  */
B200GS_API int b200gs_project_fwd(const B200gsView* view, int64_t n, const float* means, const float* scales, const float* quats,
                       const float* shs, float* xy, float* depth, int32_t* radii, float* conic, float* comp,
                       int32_t* tiles, float* cov3d, float* rgb, uint8_t* clamped, void* stream);

/* ---- K8: backward of K1 ------------------------------------------------------------------------------------------
 * in : the K1 inputs, radii (visibility), clamped (when shs), and cotangents v_xy[n,2] (vanilla: dgr's NDC-scaled
 *      dL/dmean2D, i.e. pixel gradient x (0.5W, 0.5H); gsplat: pixel units), v_depth[n] (nullable), v_conic[n,3] (true
 *      partials of power = -(A dx^2 + C dy^2)/2 - B dx dy), v_comp[n] (nullable), v_rgb[n,3] (nullable unless shs).
 * out: v_means[n,3] v_scales[n,3] v_quats[n,4] and v_shs[n,sh_stride,3] (when shs) — fully written (zeros for culled).
 * vanilla mode back-propagates the SH view direction into v_means; gsplat mode does not (renderers detach it). */
B200GS_API int b200gs_project_bwd(const B200gsView* view, int64_t n, const float* means, const float* scales, const float* quats,
                       const float* shs, const int32_t* radii, const uint8_t* clamped, const float* v_xy,
                       const float* v_depth, const float* v_conic, const float* v_comp, const float* v_rgb,
                       float* v_means, float* v_scales, float* v_quats, float* v_shs, void* stream);

/* ---- per-Gaussian passes next to the renderer in a training step (SURVEY §8f rank 4) ---------------------------------------
 * b200gs_selective_adam: visibility-masked Adam step of one [rows, width] parameter tensor (gsplat.optimizers.SelectiveAdam /
 *     diff-accel SparseGaussianAdam, internal/optimizers.py:26-90): for the rows with visible[row] != 0
 *     m = b1 m + (1-b1) g;  v = b2 v + (1-b2) g^2;  p -= lr m / (sqrt(v) + eps)   (no bias correction, like those kernels);
 *     rows that did not take part in the view keep parameter and moments untouched.
 * b200gs_densify_stats: VanillaDensityControllerImpl.update_states (vanilla_density_controller.py:101-123) in one pass: on the
 *     visible rows (visible[n] bytes, or radii > 0 when NULL) max_radii2d = max(max_radii2d, radii), grad_accum += |grad[:, :2] *
 *     (scale_x, scale_y)|, denom += 1.  grad has grad_stride floats per row (2 for gsplat xys, 3 for dgr's screenspace points). */
B200GS_API int b200gs_selective_adam(int64_t rows, int32_t width, float* param, const float* grad, float* exp_avg, float* exp_avg_sq,
                                     const uint8_t* visible, float lr, float beta1, float beta2, float eps, void* stream);
B200GS_API int b200gs_densify_stats(int64_t n, const int32_t* radii, const uint8_t* visible, const float* grad, int32_t grad_stride,
                                    float scale_x, float scale_y, float* max_radii2d, float* grad_accum, float* denom, void* stream);

/* ---- 3DGS-MCMC (internal/density_controllers/mcmc_density_controller.py) -------------------------------------------------
 * b200gs_mcmc_relocation: gsplat's compute_relocation (mcmc_density_controller.py:13,121-128), Eq. (9) of 3DGS-MCMC, one sampled
 *     Gaussian per thread.  With N = clamp(counts[i], 1, n_max):
 *         new_opacities[i] = o' = 1 - (1 - o)^(1/N)
 *         new_scales[i]    = scales[i] * o / D,   D = sum_{j=1..N} (-1)^(j-1) C(N,j) o'^j / sqrt(j)
 *     (the hockey-stick form of the paper's double sum), evaluated in fp64.  binoms is the controller's [n_max, n_max] table
 *     (mcmc_density_controller.py:53-60): it bounds N, and no entry of it is read (fp32 rounds every C(n,k) > 2^24, which
 *     moves D by up to 9e-5 relative), so unlike gsplat's kernel a count above n_max never reads outside it.
 * b200gs_mcmc_position_noise: MCMCDensityControllerImpl._add_xyz_noise (mcmc_density_controller.py:93-120) in one in-place pass
 *     over the raw parameters: means[i] += scale * w * Sigma z, Sigma = R(q) diag(s)^2 R(q)^T with s = exp(log_scales[i]) and
 *     q = raw_quats[i] / max(|raw_quats[i]|, 1e-12) (K8's fp32 geometry), o = sigmoid(opacity_logits[i]),
 *     w = 1 / (1 + exp(-100 ((1 - o) - 0.995))), and z three standard normals of Philox4x32-10 keyed by seed, subsequence
 *     offset + i.  scale = noise_lr * xyz_lr.  raw_quats must be 16-byte aligned (read as float4).
 * Algorithmic bytes: relocation 20 B in + 16 B out per sampled Gaussian; position noise 44 B in + 12 B out per Gaussian. */
B200GS_API int b200gs_mcmc_relocation(int64_t n, const float* opacities, const float* scales, const int32_t* counts, const float* binoms,
                                      int32_t n_max, float* new_opacities, float* new_scales, void* stream);
B200GS_API int b200gs_mcmc_position_noise(int64_t n, float* means, const float* log_scales, const float* raw_quats,
                                          const float* opacity_logits, float scale, uint64_t seed, uint64_t offset, void* stream);

/* ---- Bilateral-grid colour correction (internal/output_processors/bilagrid.py, internal/utils/lib_bilagrid.py) ------------------
 * b200gs_bilagrid_slice_fwd: lib_bilagrid's slice(...)["rgb"] as BilagridProcessorModule.forward calls it (bilagrid.py:115-124).
 *     grids float[n_grids,12,L,gh,gw] contiguous, xy float[batch,height,width,2] contiguous, grid_idx int64[n_idx] with n_idx == 1
 *     (one grid for every row) or n_idx == batch.  rgb and out are addressed as base[b sb + y sy + x sx + c sc] (element strides,
 *     so the processor's permuted CHW render needs no copy).  Per pixel, with G = grids[grid_idx[b]]:
 *         gray = 0.299 r + 0.587 g + 0.114 b,  ix = ((2 (x - 0.5) + 1) / 2) (gw - 1),  iy likewise with gh,
 *         iz = ((2 gray - 1 + 1) / 2) (L - 1),  each clipped to [0, size - 1];
 *         A[c] = trilinear interpolation of G[c] at (iz, iy, ix) (corners outside the grid contribute nothing),
 *         out_i = sum_j A[4i + j] rgb_j + A[4i + 3].
 *     A grid index outside [0, n_grids) reads no grid and sets that row's output to NaN.
 * b200gs_bilagrid_slice_bwd: v_out (same strides) -> v_rgb (same strides, NULL: not computed) and v_grids (accumulated into, NULL:
 *     not computed).  v_rgb includes the path through the guidance gray; a clipped coordinate passes no gradient, a coordinate
 *     exactly on 0 or size - 1 included (grid_sample's border rule).  xy gets no gradient.
 * b200gs_bilagrid_tv_fwd: lib_bilagrid's total_variation_loss (bilagrid.py:100-104) on grids float[n,channels,L,gh,gw]:
 *         tv = (1/n) sum_{axis in L,gh,gw} sum (x[.., i+1, ..] - x[.., i, ..])^2 / max(numel per grid of the difference, 1)
 *     as b200gs_bilagrid_tv_blocks(...) per-CTA partial sums, which the caller adds in a fixed order.
 * b200gs_bilagrid_tv_bwd: v_grids = v_tv[0] * d tv / d grids (v_tv a device scalar), written densely.
 * Algorithmic bytes: slice forward 8 (xy) + 12 (rgb) + 12 (out) per pixel + the grid; backward 8 + 12 + 12 (v_out) + 12 (v_rgb) per
 *     pixel + the grid and its gradient; tv forward 4 per grid element, backward 8. */
B200GS_API int b200gs_bilagrid_slice_fwd(int32_t n_grids, int32_t grid_l, int32_t grid_h, int32_t grid_w, const float* grids,
                                         int32_t batch, int32_t height, int32_t width, const float* xy, const float* rgb, int64_t sb,
                                         int64_t sy, int64_t sx, int64_t sc, const int64_t* grid_idx, int32_t n_idx, float* out,
                                         void* stream);
B200GS_API int b200gs_bilagrid_slice_bwd(int32_t n_grids, int32_t grid_l, int32_t grid_h, int32_t grid_w, const float* grids,
                                         int32_t batch, int32_t height, int32_t width, const float* xy, const float* rgb, int64_t sb,
                                         int64_t sy, int64_t sx, int64_t sc, const int64_t* grid_idx, int32_t n_idx,
                                         const float* v_out, float* v_rgb, float* v_grids, void* stream);
B200GS_API int64_t b200gs_bilagrid_tv_blocks(int32_t n, int32_t channels, int32_t grid_l, int32_t grid_h, int32_t grid_w);
B200GS_API int b200gs_bilagrid_tv_fwd(int32_t n, int32_t channels, int32_t grid_l, int32_t grid_h, int32_t grid_w, const float* grids,
                                      float* partials, void* stream);
B200GS_API int b200gs_bilagrid_tv_bwd(int32_t n, int32_t channels, int32_t grid_l, int32_t grid_h, int32_t grid_w, const float* grids,
                                      const float* v_tv, float* v_grids, void* stream);

/* ---- Appearance-embedding colour pass (internal/renderers/gsplat_appearance_embedding_renderer.py) ---------------------------------
 * The MLP of Model.forward (:77-93) and the colour / opacity epilogue of _get_rgbs_and_opacities (:239-295), on the tensor cores
 * (mma.sync TF32, each product as three TF32 products of split operands: FP32-level accuracy, FP32 accumulation).
 * B200gsAppearanceMlp (a HOST struct of sizes, flags and DEVICE pointers) describes the network:
 *     feat_dim F (a multiple of 8); n_freq: frequencies of PositionalEncoding(3, n_freq) of the view direction, < 0: no view direction;
 *     n_neurons 64 | 128; n_layers 2..4 linear layers, the output layer included; n_out 3 | 4.
 *     weights[l] / biases[l], l < n_layers: torch Linear layout [out, in].  weights[0] has w0_stride floats per row; the kernels read
 *     its columns [0, F) (features) and [w0_pe_col, w0_pe_col + 3 (2 n_freq + 1)) (view direction).  The per-image embedding is the
 *     same for every row, so the caller folds its columns into biases[0] = b_0 + W_0[:, F:F+E] e.
 *     normalize: rows of `features` are divided by max(|row|, 1e-12) first.  normalize_dirs: so is the view direction.
 *     epilogue: 0 = out[n, n_out] holds the sigmoid outputs; 1 = the renderer's colours, see below.
 * Rows: mask uint8[n] (NULL: every row); a row with mask[i] == 0 is not evaluated.  The view direction of row i is
 *     dirs[i] - cam (cam float[3] on the device, NULL: zero), both NULL when n_freq < 0.
 * b200gs_appearance_mlp_fwd, epilogue == 1, with s = the sigmoid outputs of a masked row:
 *         out[i] = clamp((base_rgb[i] + 0.5) + (2 s[0..2] - 1), 0, 1)                                    out float[n,3]
 *         n_out == 4: opacity_offsets[i] = s[3], opacities[i] = min(s[3] + raw_opacity[i], 1)
 *     and out[i] = 0, opacity_offsets[i] = 0, opacities[i] = min(raw_opacity[i], 1) for the other rows: every output is fully written.
 * b200gs_appearance_mlp_bwd: recomputes the activations.  v_out as out; v_opacities / v_opacity_offsets float[n], nullable.
 *     Writes v_base_rgb[n,3] and v_raw_opacity[n] (epilogue == 1; the latter when n_out == 4), v_features[n,F] (NULL: not computed;
 *     through the normalisation when on), each fully written with zeros in the unmasked rows, and v_params, one dense vector
 *         W_0 [n_neurons, K0p] | W_1 | .. | W_last [n_out, n_neurons] | b_0 | .. | b_last,   K0p = F + 3 (2 n_freq + 1) rounded up to 8,
 *     W_0's columns being the features, then the view direction, then zeros.  Every persistent CTA sums its rows into its own block
 *     of `workspace` (b200gs_appearance_mlp_workspace_bytes, 16-byte aligned) and a second kernel adds the blocks in a fixed order: two
 *     calls on the same inputs give bit-identical v_params.  No gradient reaches dirs or cam (the reference detaches them).
 * b200gs_appearance_mlp_workspace_bytes: 0 when the shape is not supported (sizes outside the sets above, or a first layer so wide
 *     that the weights and one 16-row tile of activations exceed 227 KB of shared memory).  A CTA runs 8 warps of 16 rows when
 *     they fit beside the weights (every 64-neuron network), else 4, 2 or 1.
 * Launches: forward 1, backward 2 (0 and 1 when n == 0), whatever the mask holds.
 * Algorithmic bytes per masked row, F = 64: forward 256 (features) + 12 + 12 (+ 12 dirs, + 4 + 8 opacity); backward 256 + 12 + 12
 *     in, 256 + 12 out.  FLOPs per masked row: 2 MACs x (K0p n_neurons + (n_layers - 2) n_neurons^2 + 8 n_neurons) forward; the
 *     backward recomputes that and adds twice as much again (gradients to the inputs and to the weights). */
#define B200GS_APPEARANCE_MAX_LAYERS 4
typedef struct B200gsAppearanceMlp {
    int32_t feat_dim, n_freq, n_neurons, n_layers, n_out;
    int32_t normalize, normalize_dirs, epilogue;
    int32_t w0_stride, w0_pe_col;
    const float* weights[B200GS_APPEARANCE_MAX_LAYERS];
    const float* biases[B200GS_APPEARANCE_MAX_LAYERS];
} B200gsAppearanceMlp;
B200GS_API size_t b200gs_appearance_mlp_workspace_bytes(int32_t feat_dim, int32_t n_freq, int32_t n_neurons, int32_t n_layers, int32_t n_out);
B200GS_API int b200gs_appearance_mlp_fwd(const B200gsAppearanceMlp* mlp, int64_t n, const float* features, const uint8_t* mask,
                                         const float* base_rgb, const float* dirs, const float* cam, const float* raw_opacity, float* out,
                                         float* opacity_offsets, float* opacities, void* stream);
B200GS_API int b200gs_appearance_mlp_bwd(const B200gsAppearanceMlp* mlp, int64_t n, const float* features, const uint8_t* mask,
                                         const float* base_rgb, const float* dirs, const float* cam, const float* raw_opacity,
                                         const float* v_out, const float* v_opacities, const float* v_opacity_offsets, float* v_base_rgb,
                                         float* v_features, float* v_raw_opacity, void* workspace, size_t workspace_bytes, float* v_params,
                                         void* stream);

/* ---- Transient visibility map (internal/renderers/gsplat_appearance_embedding_visibility_map_renderer.py, Model.visibility_forward
 *      :140-157; internal/metrics/visibility_map_metrics.py) ---------------------------------------------------------------------
 * B200gsUvGrid (host struct): tiny-cuda-nn's 2-D DenseGrid encoding, linear interpolation, 2 features per level:
 *     n_levels 1..16, base_resolution >= 1, per_level_scale >= 1.  Level l: scale_l = exp2f(l log2f(per_level_scale)) base - 1 (fp32,
 *     on the host), res_l = ceil(scale_l) + 1, size_l = res_l^2 rounded up to a multiple of 8 vertices of 2 floats; a grid is the
 *     levels in order (b200gs_uv_grid_params floats; 121760 for 8 / 16 / 1.405; a grid of more than INT32_MAX floats, or with a
 *     scale that is not finite, is not supported and gives 0).  Coordinate (u, v): pos = fmaf(scale_l, u, 0.5f),
 *     cell = floor(pos), frac = pos - cell per axis; corners k = 0..3 (bit 0: x) with weight (frac or 1 - frac in x) * (.. in y) at
 *     vertex ((cell_x + k&1) + (cell_y + k>>1) res_l) % size_l; enc[row, 2 l + f] = the weighted sum in corner order.
 * b200gs_uv_grid_fwd: enc float[n, 2 n_levels] (8-byte aligned).  uv NULL: the pixel grid of one image, n = width * height rows in
 *     row-major (y, x) order with u = x / (width - 1), v = y / (height - 1) in fp32 (width, height >= 2); else uv float[n, 2].
 *     grids: a DEVICE array of n_grids device pointers to grids; the one used is grids[*appearance_id] (int64 read on the device), or
 *     grids[host_appearance_id] when appearance_id is NULL.  An id outside [0, n_grids) reads no grid and makes enc NaN.
 * b200gs_uv_grid_bwd: v_params float[b200gs_uv_grid_params] <- the gradient of the selected grid from v_enc, written whole.  Pixel grid:
 *     one warp per vertex gathers its pixels in a fixed order (no atomics; bit-identical on every call).  uv given: float atomics.
 * Launches: forward 1 (0 when n == 0), backward 1.
 * Visibility MLP: the appearance kernels (K20-K22) with one sigmoid output and no epilogue.  mlp->feat_dim = 2 n_levels (a multiple of
 *     8), n_freq = -1, n_out = 1, normalize = normalize_dirs = epilogue = 0; the transient embedding is folded into biases[0] by the
 *     caller as for the appearance network.  out float[n]; v_enc float[n, feat_dim] (16-byte aligned, NULL: not computed); v_params
 *     as b200gs_appearance_mlp_bwd's.  b200gs_visibility_mlp_workspace_bytes: 0 for shapes the kernels do not take.
 * b200gs_vis_loss_fwd: the masked L1 + SSIM of VisibilityMapMetricsImpl.get_train_metrics on image, gt float[3, H, W], visibility
 *     float[H, W] and mask (NULL or uint8[H, W], 0 or 1), all contiguous: a' = w image, b' = w gt with w = visibility * mask, the SSIM
 *     of b200gs_loss_fwd.  Writes the derivative maps and partials[b200gs_vis_loss_blocks][3] = per-CTA sums of |a' - b'|, SSIM and
 *     (1 - visibility)^2 into the workspace (maps first, then partials; b200gs_vis_loss_workspace_bytes).  vis_grad: also the map the
 *     visibility gradient needs.
 * b200gs_vis_loss_bwd: with loss = (1 - lambda) mean|a' - b'| + lambda (1 - mean SSIM) + vis_reg_factor mean((1 - visibility)^2):
 *     v_image <- (*v_loss or 1) d loss / d image; v_visibility (NULL: not computed; needs vis_grad in the forward) <- d loss / d
 *     visibility, the three channels summed in the CTA.  Launches: forward 1, backward 1.  No atomics. */
typedef struct B200gsUvGrid {
    int32_t n_levels, base_resolution;
    float per_level_scale;
} B200gsUvGrid;
B200GS_API int64_t b200gs_uv_grid_params(const B200gsUvGrid* grid);
B200GS_API int b200gs_uv_grid_fwd(const B200gsUvGrid* grid, int32_t width, int32_t height, const float* uv, int64_t n, const float* const* grids,
                                  int32_t n_grids, const int64_t* appearance_id, int64_t host_appearance_id, float* enc, void* stream);
B200GS_API int b200gs_uv_grid_bwd(const B200gsUvGrid* grid, int32_t width, int32_t height, const float* uv, int64_t n, const float* v_enc,
                                  float* v_params, void* stream);
B200GS_API size_t b200gs_visibility_mlp_workspace_bytes(int32_t feat_dim, int32_t n_neurons, int32_t n_layers);
B200GS_API int b200gs_visibility_mlp_fwd(const B200gsAppearanceMlp* mlp, int64_t n, const float* enc, float* out, void* stream);
B200GS_API int b200gs_visibility_mlp_bwd(const B200gsAppearanceMlp* mlp, int64_t n, const float* enc, const float* v_out, float* v_enc,
                                         void* workspace, size_t workspace_bytes, float* v_params, void* stream);
B200GS_API int64_t b200gs_vis_loss_blocks(int32_t width, int32_t height);
B200GS_API size_t b200gs_vis_loss_workspace_bytes(int32_t width, int32_t height, int32_t vis_grad);
B200GS_API int b200gs_vis_loss_fwd(int32_t width, int32_t height, const float* image, const float* gt, const float* visibility,
                                   const uint8_t* mask, int32_t vis_grad, void* workspace, size_t workspace_bytes, void* stream);
B200GS_API int b200gs_vis_loss_bwd(int32_t width, int32_t height, const float* image, const float* gt, const float* visibility,
                                   const uint8_t* mask, const void* workspace, size_t workspace_bytes, float lambda_dssim,
                                   float vis_reg_factor, const float* v_loss, float* v_image, float* v_visibility, void* stream);

/* ---- Learned exposure correction (internal/output_processors/exposure.py, ExposureProcessorModule.forward :112-143) ------------
 * b200gs_exposure_fwd: one view's colour transform.  render and out are float[3,H,W] addressed as base[c sc + y sy + x sx] (element
 *     strides, so the permuted [H,W,3] render of the v1 and appearance renderers needs no copy); channels must be 3.
 *     exposure_params float[n_appearances, n_params] contiguous, n_params 4 (no bias) or 7 (with_bias); the row is the int64 read
 *     from appearance_id on the device, or host_appearance_id when appearance_id is NULL.  shade float[shade_size, shade_size]
 *     contiguous (the reference's shade_correction[0]), NULL with shade_size 0 when shade correction is off.  With
 *     a = sigmoid(exposure_params[id]):
 *         M = sigmoid(shade) / max(max(sigmoid(shade)), 1e-4),
 *         m(y, x) = F.interpolate(M, (H, W), mode="bilinear", align_corners=True)   (1 without shade correction),
 *         x_c = (a_c max_gray_scale) (render_c m) [+ 2 a_{3+c} - 1],   out_c = (clamp(x_c, 0, 1) + 1e-5) ^ (a_last max_gamma).
 *     An id outside [0, n_appearances) reads no parameter row and makes out NaN.
 * b200gs_exposure_bwd: v_out (same strides) -> v_render (same strides; the clamp passes the gradient as identity, as the reference's
 *     straight-through clamp), v_params float[n_appearances, n_params] (written whole: rows other than id are zero) and, with shade
 *     correction, v_shade float[shade_size, shade_size] (written whole; no gradient through the detached max).  Parameter sums are
 *     per-CTA partials added in a fixed order and v_shade is gathered per cell in a fixed order: two calls on the same inputs give
 *     bit-identical gradients.  An out-of-range id makes v_render NaN and v_params, v_shade zero.
 * b200gs_exposure_workspace_bytes: device scratch of the forward (backward == 0) or the backward (backward != 0) at this image and
 *     shade size; 0 for sizes the kernels do not take (H or W < 1, H > 524280, H W > 2^31 - 1, shade_size outside 0..4096).
 * Launches: forward 2 (prologue, pixels), backward 3 (prologue, pixels, reduction).  No host synchronisation.
 * Algorithmic bytes: forward 12 in + 12 out per pixel; backward 24 in + 12 out per pixel, plus, with shade correction, v_m 4 out and
 *     4 in per pixel. */
B200GS_API size_t b200gs_exposure_workspace_bytes(int32_t height, int32_t width, int32_t shade_size, int32_t backward);
B200GS_API int b200gs_exposure_fwd(int32_t channels, int32_t height, int32_t width, const float* render, int64_t sc, int64_t sy, int64_t sx,
                                   int32_t n_appearances, int32_t n_params, const float* exposure_params, const int64_t* appearance_id,
                                   int64_t host_appearance_id, int32_t shade_size, const float* shade, float max_gray_scale,
                                   float max_gamma, void* workspace, size_t workspace_bytes, float* out, void* stream);
B200GS_API int b200gs_exposure_bwd(int32_t channels, int32_t height, int32_t width, const float* render, int64_t sc, int64_t sy, int64_t sx,
                                   int32_t n_appearances, int32_t n_params, const float* exposure_params, const int64_t* appearance_id,
                                   int64_t host_appearance_id, int32_t shade_size, const float* shade, float max_gray_scale,
                                   float max_gamma, void* workspace, size_t workspace_bytes, const float* v_out, float* v_render,
                                   float* v_params, float* v_shade, void* stream);

/* ---- Inverse-depth regularisation (internal/metrics/inverse_depth_metrics.py:70-107, get_inverse_depth_metric) -------------------
 * b200gs_depth_loss_fwd: pred (the rendered inverse depth) and gt float[height, width] contiguous; mask NULL or a uint8 keep-mask
 *     read at mask[mask_sy y + mask_sx x] (channel 0 of the reference's [C,H,W] image mask, no copy; nonzero keeps the pixel).
 *     norm 0: none; 1: pred' = (pred - min) / (max - min + 1e-8) over the whole pred; 2: pred' = pred / median; 3: m = mean(gt),
 *     gt' = gt / m, pred' = pred / m.  a = gt' k, b = pred' k with k the mask (1 without one).  loss_type 0: mean|a - b|;
 *     1: mean (a - b)^2; 2 (no mask, height and width >= 11): (1 - ssim_weight) mean|a - b| + ssim_weight (1 - SSIM), SSIM being
 *     torchmetrics' StructuralSimilarityIndexMeasure() (11-tap Gaussian, sigma 1.5, data range max(range(a), range(b)),
 *     C1 = (0.01 dr)^2, C2 = (0.03 dr)^2, reflect pad and 5-pixel crop = the mean over the (H-10)(W-10) full-window positions).
 *     Writes loss[0] and stats[0..1] = [mean |a - b| or (a - b)^2, mean SSIM (NaN for loss types 0 and 1)] on the device.
 * b200gs_depth_loss_bwd: v_pred float[height, width] <- (*v_loss or 1) d loss / d pred, including the gradient through the data
 *     range into b's extremum pixels (split evenly among tied pixels; half of it when the two ranges tie).  gt has no gradient.
 *     It reads the workspace its forward wrote, with the same arguments.  All sums are per-CTA partials added in a fixed order:
 *     two calls give bit-identical results.
 * b200gs_depth_loss_workspace_bytes: device scratch shared by the forward and the backward; 0 for sizes the kernels do not take
 *     (height or width < 1, height > 1048560, height width > 2^31 - 1, loss_type outside 0..2).
 * Launches: forward 4 (statistics, prologue, tiles, loss), backward 1.  No host synchronisation.
 * Algorithmic bytes: forward 8 in per pixel (the tiles read pred and gt), + 8 when the statistics pass runs (l1+ssim, norm 1 or
 *     3), + 1 with a mask, + 12 out with SSIM (the three derivative maps); backward 8 in + 4 out per pixel (+ 1 with a mask, + 12 in with SSIM). */
B200GS_API size_t b200gs_depth_loss_workspace_bytes(int32_t height, int32_t width, int32_t loss_type);
B200GS_API int b200gs_depth_loss_fwd(int32_t height, int32_t width, const float* pred, const float* gt, const uint8_t* mask,
                                     int64_t mask_sy, int64_t mask_sx, int32_t loss_type, int32_t norm, float median, float ssim_weight,
                                     void* workspace, size_t workspace_bytes, float* loss, float* stats, void* stream);
B200GS_API int b200gs_depth_loss_bwd(int32_t height, int32_t width, const float* pred, const float* gt, const uint8_t* mask,
                                     int64_t mask_sy, int64_t mask_sx, int32_t loss_type, int32_t norm, float median, float ssim_weight,
                                     const void* workspace, size_t workspace_bytes, const float* v_loss, float* v_pred, void* stream);

/* ---- Gaussian regularisers (internal/metrics/mcmc_metrics.py:39-59, MCMCMetricsModuleMixin.reg_loss, and
 *      internal/metrics/scale_regularization_metrics.py:51-115, get_scale_regularization_metrics) --------------------------------
 * b200gs_gaussian_reg_fwd: opacities float[n,1] and scales float[n,3] contiguous: with B200GS_GREG_RAW the logits and log-scales
 *     (activated here as torch's fp32 sigmoid and exp), otherwise the activated values (get_opacity / get_scales()).  Writes
 *     terms[0..3] = [opacity_weight mean|o|                                         (mcmc_metrics.py:42, flag OPACITY)
 *                    scale_weight mean|s|                                           (mcmc_metrics.py:46, flag SCALE)
 *                    scale_lambda sum(s [s > max_scale]) / (n_s + 1)                 (scale_regularization_metrics.py:74-82, OVER_SCALE)
 *                    ratio_lambda sum(r [r > max_scale_ratio]) / (n_r + 1)]          (scale_regularization_metrics.py:84-90, OVER_RATIO)
 *     with n_s = #{s > max_scale} elementwise, r = max / (mid + 1e-8) of each row sorted ascending (tied values routed as torch.sort
 *     routes them on the GPU, a table measured on an H100: it decides which column takes the "mid" gradient), both thresholds strict.  A term whose flag is clear or whose weight is 0 is 0.  stats NULL
 *     or float[5] <- [n_s, n_r, max of the largest scale, max r, mean r] (scale_regularization_metrics.py:92-98; n_s / n_r are 0
 *     when their term is off).  opacities may be NULL when OPACITY is clear, scales when no scale flag is set and stats is NULL.
 * b200gs_gaussian_reg_bwd: v_opacities float[n,1] (when opacities is given) and v_scales float[n,3] (when scales is given) <-
 *     sum_k v_terms[k] d terms[k] / d input, dense, exact zeros wherever no term applies (torch.abs' subgradient at 0 is 0); with
 *     RAW chained through the activations as torch does (y (1 - y) and y from the fp32 output).  v_terms float[4] is read on the
 *     device.  It reads the coefficients its forward wrote to the workspace, and takes the same arguments.  No float atomics: two
 *     calls give bit-identical results.
 * b200gs_gaussian_reg_workspace_bytes: device scratch shared by the forward and the backward; 0 for n < 1 or n > 2^31 - 1.
 * Launches: forward 2 (per-CTA partials, reduce), backward 1.  No host synchronisation.
 * Algorithmic bytes: forward 16 in per Gaussian (4 without the scale terms and statistics, 12 without the opacity term); backward
 *     16 in + 16 out per Gaussian. */
#define B200GS_GREG_RAW 1
#define B200GS_GREG_OPACITY 2
#define B200GS_GREG_SCALE 4
#define B200GS_GREG_OVER_SCALE 8
#define B200GS_GREG_OVER_RATIO 16
B200GS_API size_t b200gs_gaussian_reg_workspace_bytes(int64_t n);
B200GS_API int b200gs_gaussian_reg_fwd(int64_t n, const float* opacities, const float* scales, int32_t flags, float opacity_weight,
                                       float scale_weight, float max_scale, float max_scale_ratio, float scale_lambda, float ratio_lambda,
                                       void* workspace, size_t workspace_bytes, float* terms, float* stats, void* stream);
B200GS_API int b200gs_gaussian_reg_bwd(int64_t n, const float* opacities, const float* scales, int32_t flags, float opacity_weight,
                                       float scale_weight, float max_scale, float max_scale_ratio, float scale_lambda, float ratio_lambda,
                                       const void* workspace, size_t workspace_bytes, const float* v_terms, float* v_opacities,
                                       float* v_scales, void* stream);

/* ---- Depth-normal consistency (internal/metrics/normal_reg.py:27-38, NormalRegModuleMixin.get_normal_reg_metrics, and gsplat's
 *      utils.depth_to_normal as it calls it) ---------------------------------------------------------------------------------------
 * n_d[y,x] = alpha[y,x] normalize(cross(p[y+1,x] - p[y-1,x], p[y,x+1] - p[y,x-1])) with p[y,x] = o + depth[y,x] R ((x - cx + 0.5) / fx,
 *     (y - cy + 0.5) / fy, 1), R / o the camera-to-world rotation / origin, normalize dividing by max(|v|, 1e-12); 0 on the one-pixel
 *     border (everywhere when height or width < 3).  The origin cancels and is never formed (exact in real arithmetic; in fp32 it
 *     avoids the reference's cancellation at large camera translations).  Every entry point computes n_d with the same code, so the
 *     forward, the backward and depth_to_normal agree bit for bit.
 * Matrices are read on the device, never copied to the host: the 4x4 camera matrix at m[i s0 + j s1] (only its 3x3 block is read) and
 *     K float[3,3] at K[i K_s0 + j K_s1] (fx = K[0,0], fy = K[1,1], cx = K[0,2], cy = K[1,2]).
 * b200gs_normal_reg_fwd: normal float[3,H,W] at normal[c normal_sc + y normal_sy + x normal_sx] (a channel slice of the permuted
 *     render, read in place), depth and alpha float[H,W] contiguous, w2c the world-to-camera matrix (normal_reg.py:29-31 inverts it
 *     with torch.linalg.inv, which synchronises; here the 3x3 block is inverted in double once per CTA, equal to the 3x3 block of
 *     the inverse for an affine [R t; 0 1]).  loss float[1] <- weight mean_{H W}(1 - sum_c normal[c] n_d[c]) (normal_reg.py:31-35,
 *     err * normal_reg_lambda).
 * b200gs_normal_reg_bwd: v_normal float[3,H,W] contiguous <- -v_loss[0] weight / (H W) n_d, v_loss read on the device; it reads the
 *     coefficient its forward wrote to the workspace and takes the same depth, alpha and matrices.
 * b200gs_depth_to_normal: normals float[H,W,3] contiguous <- n_d with alpha = 1 from depth float[H,W] contiguous and c2w the
 *     camera-to-world matrix (gsplat utils.depth_to_normal with z_depth = True, normal_reg.py:29-32).
 * b200gs_normal_reg_workspace_bytes: device scratch shared by the forward and the backward; 0 for a size that is not accepted.
 * Sizes: 1 <= height <= 65535 * 16, width >= 1, height * width <= 2^31 - 1.
 * Launches: forward 2 (per-tile partials, reduce), backward 1, depth_to_normal 1.  No host synchronisation, no float atomics: two
 *     calls give bit-identical results.
 * Algorithmic bytes per pixel: forward 4 depth + 4 alpha + 12 normal in; backward 8 in + 12 out; depth_to_normal 4 in + 12 out. */
B200GS_API size_t b200gs_normal_reg_workspace_bytes(int32_t height, int32_t width);
B200GS_API int b200gs_normal_reg_fwd(int32_t height, int32_t width, const float* normal, int64_t normal_sc, int64_t normal_sy,
                                     int64_t normal_sx, const float* depth, const float* alpha, const float* w2c, int64_t w2c_s0,
                                     int64_t w2c_s1, const float* K, int64_t K_s0, int64_t K_s1, float weight, void* workspace,
                                     size_t workspace_bytes, float* loss, void* stream);
B200GS_API int b200gs_normal_reg_bwd(int32_t height, int32_t width, const float* depth, const float* alpha, const float* w2c, int64_t w2c_s0,
                                     int64_t w2c_s1, const float* K, int64_t K_s0, int64_t K_s1, const void* workspace,
                                     size_t workspace_bytes, const float* v_loss, float* v_normal, void* stream);
B200GS_API int b200gs_depth_to_normal(int32_t height, int32_t width, const float* depth, const float* c2w, int64_t c2w_s0, int64_t c2w_s1,
                                      const float* K, int64_t K_s0, int64_t K_s1, float* normals, void* stream);

/* ---- k nearest neighbours on a hash grid over the reference points (no host synchronisation: the grid is sized on the device) ----
 * b200gs_knn_mean_dist2: simple_knn's distCUDA2 (vanilla_gaussian.py:122-125, the scale initialiser): mean_dist2[i] = mean of the squared
 *     distances from points[i] (float[n,3]) to its 3 nearest neighbours (exact).
 * b200gs_knn_points: pytorch3d.ops.knn_points for one batch entry with norm 2 and sorted output (appearance_feature_similarity_
 *     regularization_metrics.py:70-74, segany_splatting.py:276-280): for every query (float[s,3]; inside or outside the reference set's
 *     bounding box) the k nearest of the n reference points (float[n,3]), a query that is itself a reference point included, in
 *     ascending order: dists float[s,k] squared fp32 distances, idx int64[s,k].  Exact up to ties: points at the same distance keep the
 *     grid's order.  Points with a non-finite coordinate are left out of the grid's bounding box; a query with fewer than k points at
 *     a finite distance (a NaN or infinite query, non-finite points) fills its remaining slots with the lowest unused indices and
 *     their distances as computed, so every index is in [0, n).  The grid sizing runs a bounded number of steps on any box.  B200GS_EINVAL for k outside 1..32 or k > n, B200GS_ENOSPACE for n >= 2^30 or a short workspace.
 * b200gs_knn_workspace_bytes: the workspace of both for n reference points.
 * Launches: 6 + ceil(log2(4n + 64) / 8) (bounds, grid, cell keys, histogram, the radix passes, gather, search).  No float atomics. */
B200GS_API size_t b200gs_knn_workspace_bytes(int64_t n);
B200GS_API int b200gs_knn_mean_dist2(int64_t n, const float* points, float* mean_dist2, void* workspace, size_t workspace_bytes, void* stream);
B200GS_API int b200gs_knn_points(int64_t s, const float* queries, int64_t n, const float* points, int32_t k, float* dists, int64_t* idx,
                                 void* workspace, size_t workspace_bytes, void* stream);

/* ---- Appearance-feature similarity regulariser (appearance_feature_similarity_regularization_metrics.py:63-102,
 *      SimilarityRegularizationMixin.get_similarity_metric after knn_points, and its autograd backward) ------------------------------
 * out float[2] <- [lambda m, m],  m = mean_{s, i<j} r_sij w_sj  over the S K (K - 1) / 2 pairs,  w_sj = exp(-decay dists[s,j]);
 *     kind 0 (Cosine): r_sij = -n_i . n_j with n = f / max(|f|, 1e-12) (F.normalize); kind 1 (Euclidean): r_sij = |f_i - f_j|;
 *     f_i = features[idx[s,i]] (features float[n,d] contiguous, idx int64[s,k] with values in [0, n), dists float[s,k]); an index
 *     outside [0, n) is clamped into it, so it reads a real row (memory-safe, not meaningful).
 *     weights float[s,k] <- w when not NULL.
 * b200gs_similarity_reg_bwd: v_features float[n,d] (every row written, 0 where no sample reached) <- d (v_loss[0] out[0]) / d features,
 *     v_loss read on the device; dists get no gradient.  Zero-norm rows take F.normalize's 1/eps branch, zero distances torch's zero
 *     norm gradient.  Per-entry rows are sorted by idx (onesweep) and summed per Gaussian in entry order: no float atomics, repeats
 *     are bit-identical.
 * Sizes: 1 <= d <= 256, 2 <= k <= 32, s >= 1, n >= 1, n < 2^30, s k < 2^30; kind 0 or 1; B200GS_EINVAL otherwise, before any CUDA call.
 * b200gs_similarity_reg_workspace_bytes: scratch of the forward (backward 0: the s per-sample sums) or of the backward (backward 1:
 *     s k (4 d + 16) bytes of entry rows and records, n 8 bytes of run table and the sort's counters); 0 for sizes not accepted.
 *     The two calls need not share a workspace: the backward reads nothing the forward wrote.
 * Launches: forward 2 (per-sample sums, reduce); backward 4 + ceil(log2(n) / 8) (entries, histogram, radix passes, run table,
 *     per-Gaussian sums). */
B200GS_API size_t b200gs_similarity_reg_workspace_bytes(int64_t n, int64_t s, int32_t k, int32_t d, int32_t backward);
B200GS_API int b200gs_similarity_reg_fwd(int64_t n, int32_t d, const float* features, int64_t s, int32_t k, const int64_t* idx,
                                         const float* dists, int32_t kind, float decay, float lambda, void* workspace,
                                         size_t workspace_bytes, float* out, float* weights, void* stream);
B200GS_API int b200gs_similarity_reg_bwd(int64_t n, int32_t d, const float* features, int64_t s, int32_t k, const int64_t* idx,
                                         const float* dists, int32_t kind, float decay, float lambda, void* workspace,
                                         size_t workspace_bytes, const float* v_loss, float* v_features, void* stream);

/* ---- standalone SH (gsplat.sh.spherical_harmonics; gsplat_renderer.py:105) -------------------------------------------
 * dirs[n,3] need not be unit (normalised inside, as gsplat does).  out rgb[n,3] = SH (no +0.5, no clamp).
 * bwd: v_coeffs[n,sh_stride,3] fully written; v_dirs[n,3] nullable. */
B200GS_API int b200gs_sh_fwd(int32_t degree, int32_t sh_stride, int64_t n, const float* dirs, const float* coeffs, float* rgb, void* stream);
B200GS_API int b200gs_sh_bwd(int32_t degree, int32_t sh_stride, int64_t n, const float* dirs, const float* coeffs, const float* v_rgb,
                  float* v_coeffs, float* v_dirs, void* stream);

/* ---- split, masked SH (spherical_harmonics_decomposed of yzslab's gsplat fork) ------------------------------------------
 * Call sites: gsplat_v1_renderer.py:124 (separate_sh), gsplat_appearance_embedding_renderer.py:193,208, glossy_renderer.py:21,
 * gsplat_distributed_renderer.py:419.  The coefficients are dc[n,1,3] | rest[n,k_rest,3] read in place (no concatenation);
 * sh_stride = 1 + k_rest >= (degree+1)^2, rest may be NULL when k_rest = 0.  mask[n] (uint8, nullable): a row with mask[i] == 0
 * reads no coefficient and gets rgb = 0 and zero v_dc / v_rest / v_dirs.  The same kernels as b200gs_sh_fwd / _bwd with another
 * coefficient loader: unmasked rows are bit-identical to those on the concatenated tensor.
 * bwd: v_dc[n,1,3] and v_rest[n,k_rest,3] fully written; v_dirs[n,3] nullable.
 * Algorithmic bytes per unmasked row at degree 3: fwd 12 + 192 in, 12 out; bwd 24 + 192 in (v_dirs), 192 out (+12). */
B200GS_API int b200gs_sh_split_fwd(int32_t degree, int32_t k_rest, int64_t n, const float* dirs, const float* dc, const float* rest,
                                   const uint8_t* mask, float* rgb, void* stream);
B200GS_API int b200gs_sh_split_bwd(int32_t degree, int32_t k_rest, int64_t n, const float* dirs, const float* dc, const float* rest,
                                   const uint8_t* mask, const float* v_rgb, float* v_dc, float* v_rest, float* v_dirs, void* stream);

/* ---- K47 / K48: Glossy-Gaussian view-dependent opacity and SH colour (glossy_renderer.py get_opacities / get_rgbs with
 *      GlossyGaussianModel.get_view_dep_opacities, glossy_gaussian.py:66-79) --------------------------------------------------
 * dir_i = (means[i] - campos) / max(|means[i] - campos|, 1e-12) (F.normalize; a Gaussian at the camera centre gets the zero
 *     direction); means float[n,3], campos float[3] on the device (never read on the host).
 * opacity[i] = clamp(SH_degree(op_dc[i] | op_rest[i]; dir_i) + 0.5, 0, 1) for EVERY row: op_dc float[n] (the [n,1,1] property),
 *     op_rest float[n,op_k_rest] (the [n,R,1] property), op_k_rest + 1 >= (degree+1)^2; rows at or beyond the degree are not read.
 * rgb[i,3] (nullable: no colour) = clamp(SH_degree(colour; dir_i) + 0.5, min=0) where mask[i] != 0 (mask uint8[n], nullable = all),
 *     0.5 elsewhere, reading no colour coefficient.  Colour: sh_split = 1: shs = dc [n,1,3], shs_rest = rest [n,sh_stride-1,3];
 *     sh_split = 0: shs = [n,sh_stride,3]; sh_stride >= (degree+1)^2.
 * clamped uint8[n] <- the clamp decisions the backward needs (bit c: colour channel c clamped or the row masked; bit 3: opacity
 *     clamped).  Bounds are inclusive as in torch.clamp: a value exactly on a bound passes its gradient.
 * bwd: v_op_dc float[n], v_op_rest float[n,op_k_rest] and, when v_rgb (float[n,3]) is not NULL, v_shs / v_shs_rest in the forward's
 *     colour layout, every row written in full: zeros at or beyond the degree, on masked rows and for clamped outputs.  No means or
 *     direction gradient (the reference detaches the direction), no coefficient read, no atomics: repeats are bit-identical.
 * degree 0..4, n >= 0; B200GS_EINVAL before any CUDA call otherwise.  Launches: one each way, no host synchronisation.
 * Algorithmic bytes per Gaussian at degree 3 (16-coefficient storage): fwd 269 in, 17 out; bwd 29 in, 256 out. */
B200GS_API int b200gs_glossy_sh_fwd(int32_t degree, int64_t n, const float* means, const float* campos, const float* op_dc,
                                    const float* op_rest, int32_t op_k_rest, const float* shs, const float* shs_rest, int32_t sh_stride,
                                    int32_t sh_split, const uint8_t* mask, float* opacity, float* rgb, uint8_t* clamped, void* stream);
B200GS_API int b200gs_glossy_sh_bwd(int32_t degree, int64_t n, const float* means, const float* campos, int32_t op_k_rest,
                                    int32_t sh_stride, int32_t sh_split, const uint8_t* clamped, const float* v_opacity,
                                    const float* v_rgb, float* v_op_dc, float* v_op_rest, float* v_shs, float* v_shs_rest, void* stream);

/* ---- K49 / K50 and the SWAG MLP: in-the-wild appearance of SWAGRenderer.forward (swag_renderer.py:32-66, swag_model.py) ---------
 * B200gsHashGrid (host struct): tiny-cuda-nn's 3-D HashGrid encoding, linear interpolation: n_levels 1..16, n_features_per_level
 *     F = 2 | 4, log2_hashmap_size 1..24, base_resolution >= 1, per_level_scale >= 1.  Level l (fp32, on the host): scale_l =
 *     exp2f(l log2f(per_level_scale)) base - 1 (< 2^30), res_l = ceil(scale_l) + 1, size_l = min(next_multiple(res_l^3, 8),
 *     2^log2_hashmap_size) vertices of F floats, the levels in order: b200gs_hash_grid_params floats (11681792 for 8 / 4 / 19 / 16 /
 *     2.0; 0 for a grid outside that set).  Point x: pos = fmaf(scale_l, x, 0.5f), cell = (uint32)(int)floor(pos), frac = pos -
 *     floor(pos) per axis; corner k = 0..7 (bit d: axis d) weighs prod_d (bit ? frac_d : 1 - frac_d) and reads vertex tcnn
 *     grid_index(cell + bits) (dense strides while they fit size_l, else the coherent prime hash 1 / 2654435761 / 805459861 xor-ed)
 *     % size_l.  Points outside [0, 1] follow the same uint32 arithmetic.
 * b200gs_swag_inputs_fwd (K49): x0 float[n, row_stride] <- [rgb | enc | 0 ..], row_stride <= 72.  With shs (colour on):
 *     rgb = clamp_min(SH_degree(colour; dir_i) + 0.5, 0), dir_i = (means[i] - campos) / max(|.|, 1e-12), colour sh_split = 1:
 *     shs = dc [n,1,3], shs_rest = rest [n,sh_stride-1,3]; sh_split = 0: shs = [n,sh_stride,3]; sh_stride >= (degree+1)^2, degree 0..4;
 *     clamped uint8[n] <- bit c set where channel c failed x >= 0 (NaN included).  shs NULL: no colour columns, enc from column 0.
 *     enc = the grid of table float[b200gs_hash_grid_params] (aligned to one vertex) at (means[i] - bbox[0..2]) / bbox[3..5]
 *     (IEEE division; bbox float[6] on the device, NULL: means[i] itself).
 * b200gs_swag_inputs_bwd (K50): from v_x0 float[n, row_stride]: colour on: v_shs (and v_shs_rest) in the forward's layout, every
 *     row written in full, and v_means float[n,3] through the view direction, after the clamp bits; v_table float[params] zeroed
 *     here and then accumulated with vector float atomics (one per corner): not bit-reproducible.  Pad columns are not read.
 * Launches: K49 1, K50 1 (0 when n == 0) and one cudaMemsetAsync.
 * Algorithmic bytes per Gaussian, degree 3, default grid, row_stride 40: fwd 204 in + 161 out + 64 gathers of 16 B; bwd 365 in +
 *     204 out + 64 vector atomics of 16 B.  FLOPs: ~900 fwd, ~1300 bwd (SH basis and gradient, 64 weights and corner indices).
 * SWAG MLP (K20/K21 with epilogue 2): mlp as for b200gs_appearance_mlp_* with n_freq = -1, n_out = 4, normalize = normalize_dirs = 0,
 *     epilogue = 2; feat_dim = row_stride of x0, in_dim the real columns (feat_dim - 8 < in_dim <= feat_dim): the kernels read W_0's
 *     columns [0, in_dim) and treat [in_dim, feat_dim) as zero, so the caller may pass the reference's [n_neurons, in_dim + E] W_0
 *     (w0_stride >= in_dim) with the image embedding folded into biases[0].  With o the 4 outputs of a row and u (float[1] on the
 *     device, in (0, 1) or 0.5 in evaluation):
 *         colour[i] = sigmoid(o[0..2]),  z = float(1 / temperature) ((log(|o3| + eps) + log(u + eps)) - log(1 - u + eps)),
 *         opacity[i] = clamp_min(base_opacity[i] - sigmoid(z), 0)                      base_opacity float[n] (activated)
 *     bwd: torch's rules (abs has gradient 0 at 0; clamp_min passes where its argument >= 0); v_colour float[n,3] and v_opacity float[n]
 *     (nullable: zero); writes v_x0 float[n, feat_dim] (16-byte aligned), v_base_opacity float[n] and v_params as
 *     b200gs_appearance_mlp_bwd's (W_0's block [n_neurons, feat_dim]; columns at or past in_dim are zero).  temperature > 0, eps >= 0.
 * Launches: forward 1, backward 2.  Bytes per row: fwd 4 feat_dim + 4 in, 16 out; bwd 4 feat_dim + 20 in, 4 feat_dim + 4 out.
 *     FLOPs per row: 2 x (feat_dim n_neurons + (n_layers - 2) n_neurons^2 + 8 n_neurons) forward (~13 K for the defaults), three
 *     times that backward. */
typedef struct B200gsHashGrid {
    int32_t n_levels, n_features_per_level, log2_hashmap_size, base_resolution;
    float per_level_scale;
} B200gsHashGrid;
B200GS_API int64_t b200gs_hash_grid_params(const B200gsHashGrid* grid);
B200GS_API int b200gs_swag_inputs_fwd(const B200gsHashGrid* grid, int32_t degree, int64_t n, const float* means, const float* campos,
                                      const float* shs, const float* shs_rest, int32_t sh_stride, int32_t sh_split, const float* bbox,
                                      const float* table, int32_t row_stride, float* x0, uint8_t* clamped, void* stream);
B200GS_API int b200gs_swag_inputs_bwd(const B200gsHashGrid* grid, int32_t degree, int64_t n, const float* means, const float* campos,
                                      const float* shs, const float* shs_rest, int32_t sh_stride, int32_t sh_split, const float* bbox,
                                      const uint8_t* clamped, const float* v_x0, int32_t row_stride, float* v_shs, float* v_shs_rest,
                                      float* v_means, float* v_table, void* stream);
B200GS_API size_t b200gs_swag_mlp_workspace_bytes(int32_t feat_dim, int32_t n_neurons, int32_t n_layers);
B200GS_API int b200gs_swag_mlp_fwd(const B200gsAppearanceMlp* mlp, int32_t in_dim, int64_t n, const float* x0, const float* base_opacity,
                                   const float* u, float temperature, float eps, float* colour, float* opacity, void* stream);
B200GS_API int b200gs_swag_mlp_bwd(const B200gsAppearanceMlp* mlp, int32_t in_dim, int64_t n, const float* x0, const float* base_opacity,
                                   const float* u, float temperature, float eps, const float* v_colour, const float* v_opacity,
                                   float* v_x0, float* v_base_opacity, void* workspace, size_t workspace_bytes, float* v_params,
                                   void* stream);

/* ---- K51 / K52: 4DGS deformation of VanillaGS4DRenderer.forward (vanilla_gs4d_renderer.py, gs4d_deformation.py, gs4d_hexplane.py) --
 * Forward only (the reference renders trained 4DGaussians checkpoints and never trains this network).
 * B200gsGs4d (host struct): the HexPlane field and the network.  n_levels L 1..4, channels C (output_coordinate_dim) 16 | 32,
 *     net_width W 64 | 128, defor_depth D 0..2 (0 and 1: one trunk Linear), flags any of B200GS_GS4D_*; resolution[l] = (x, y, z, t)
 *     nodes of level l, each 1..B200GS_GS4D_MAX_RES, every plane below 2^31 floats.  Plane k = (a, b) of (0,1), (0,2), (0,3), (1,2),
 *     (1,3), (2,3) is [C, res_b, res_a] in torch (coordinate a indexes the width).  weights[i] [rows, K] row-major (16-byte aligned)
 *     and biases[i] [rows], as torch.nn.Linear holds them: i = 0 the trunk's first Linear [W, C L], 1 its second [W, W] (D = 2
 *     only), then for head h = 0 dx, 1 ds, 2 dr, 3 dshs: 2 + 2h its hidden Linear [W, W] and 3 + 2h its output Linear [3 | 3 | 4 |
 *     48, W].  Pointers of layers not in use are not read.
 * b200gs_gs4d_plane_floats: floats of the repacked planes (the buffer b200gs_gs4d_repack_planes fills); 0 for a grid or network
 *     outside the supported set.  No CUDA call: it is also the support query.
 * b200gs_gs4d_repack_planes (K52): host_planes = 6 L device pointers (level-major, then plane order) to the torch planes; writes
 *     planes float[b200gs_gs4d_plane_floats] channel-last: each plane [res_b, res_a, C], at the plane's offset in that order.
 * b200gs_gs4d_deform_fwd (K51): n Gaussians (0 <= n <= INT32_MAX), all device pointers: aabb float[6] = (xyz_max, xyz_min) as the
 *     reference's set_aabb stores it, time float[1] (t as given), means / log_scales float[n,3] and quats float[n,4] (raw, 16-byte
 *     aligned), shs_dc float[n,1,3] and shs_rest float[n,15,3] (read with B200GS_GS4D_DSHS only).  With p = (means - xyz_max) *
 *     (2 / (xyz_min - xyz_max)) - 1 (fp32, IEEE, not clamped) and f = the levels' products of the six bilinear plane samples of
 *     (p, t) (align_corners, border padding, in plane order from 1), h = the trunk on f with ReLU between its layers, and each
 *     enabled head Linear relu Linear relu h:
 *         means_out = means + dx,  log_scales_out = log_scales + ds,  quats_out = quats + dr (B200GS_GS4D_APPLY_ROTATION: the
 *         Hamilton product quats dr divided by its norm),  shs_*_out = shs_* + dshs reshaped [16, 3]
 *     A disabled dx / ds / dr head copies its input to the output; with dshs off the SH outputs are not written (may be NULL).
 *     Weights run as 3xTF32 mma.sync with fp32 accumulation (~fp32 accuracy).  No workspace; launches: one.  Bytes per Gaussian:
 *     40 in + 40 out (+ 192 in + 192 out with dshs) plus 24 L corner rows of 4 C bytes gathered; FLOPs per Gaussian 2 (C L W +
 *     (D' - 1) W^2 + sum over enabled heads (W^2 + W out_h)).
 * Both refuse with B200GS_EINVAL before any CUDA call. */
#define B200GS_GS4D_DX 1
#define B200GS_GS4D_DS 2
#define B200GS_GS4D_DR 4
#define B200GS_GS4D_DSHS 8
#define B200GS_GS4D_APPLY_ROTATION 16
#define B200GS_GS4D_FLAGS 31
#define B200GS_GS4D_MAX_RES 16384
typedef struct B200gsGs4d {
    int32_t n_levels, channels, net_width, defor_depth, flags;
    int32_t resolution[4][4];
    const float* weights[10];
    const float* biases[10];
} B200gsGs4d;
B200GS_API int64_t b200gs_gs4d_plane_floats(const B200gsGs4d* grid);
B200GS_API int b200gs_gs4d_repack_planes(const B200gsGs4d* grid, const float* const* host_planes, float* planes, void* stream);
B200GS_API int b200gs_gs4d_deform_fwd(const B200gsGs4d* grid, int64_t n, const float* planes, const float* aabb, const float* time,
                                      const float* means, const float* log_scales, const float* quats, const float* shs_dc,
                                      const float* shs_rest, float* means_out, float* log_scales_out, float* quats_out,
                                      float* shs_dc_out, float* shs_rest_out, void* stream);

/* ---- K2-K5: tile binning ------------------------------------------------------------------------------------------
 * replaces dgr InclusiveSum + duplicateWithKeys + SortPairs + identifyTileRanges / gsplat isect_tiles + isect_offset_encode.
 * Result order is exactly that of a stable sort of (tile_id << 32 | float_bits(depth)) keys emitted Gaussian-major:
 * implemented as a stable depth sort of the visible Gaussians, a stable partition of (coarse cell, Gaussian) pairs (a
 * cell = 8x8 tiles) and an order-preserving multi-split of every cell's list into its 64 tiles that writes each id
 * once.  Both sorts are hand-written onesweep-style radix passes (decoupled look-back); no library sort is involved.
 *
 * Counters: d_counts = device int64[4], host_counts = host int64[4] (pinned or pageable; nullable):
 *     [0] number of (tile, Gaussian) pairs of the 3-sigma bounding rects — the reference's pair count, an upper bound
 *         of [2] and equal to it without culling                                              (written by phase A)
 *     [1] number of (coarse cell, Gaussian) pairs                                              (written by phase A)
 *     [2] number of pairs actually listed in sorted_ids / tile_ranges                          (written by phase B)
 *     [3] number of visible Gaussians (non-empty tile rect)                                    (written by phase A)
 *   Each phase ends by delivering d_counts to host_counts (when != NULL) in stream order — pinned/mapped host memory is
 *   written by a tiny kernel with system-scope stores (a D2H copy would queue on a copy engine behind the application's
 *   bulk transfers), pageable memory by cudaMemcpyAsync — and, when sync_host != 0, SYNCHRONISES the stream.
 *   Sync-free use: size max_coarse from the previous view's counts[1] and max_pairs from its counts[0] (the bound is known
 *   after phase A already), pass sync_host = 0, record an event after phase A and check
 *   counts[1] <= max_coarse && counts[0] <= max_pairs once the rest of the forward has been enqueued.
 * cull_conic[n,3] / cull_opacity[n] (both NULL, or both given): exact tile culling.  A (tile, Gaussian) pair is dropped
 *     when no pixel sample of the tile can reach alpha >= 1/255 for that Gaussian (minimum of the conic's quadratic
 *     over the tile box > ln(255*opacity)); the blend loop would have skipped it at every pixel, so images and
 *     gradients do not change while the pair list shrinks ~2x.  With NULL the pair list is exactly the reference's
 *     (every tile of the 3-sigma bounding rect).
 * b200gs_bin_count_workspace_bytes / b200gs_bin_sort_workspace_bytes: bytes of scratch for phase A (n Gaussians) and
 *     phase B (up to max_coarse coarse pairs).  Two buffers because counts[1] is only known after phase A.
 * b200gs_bin_count: phase A.  Compaction of the visible Gaussians, depth keys, stable depth sort; counts[0], [1], [3].  Everything
 *     phase B needs to know about a Gaussian (xy, radius, cull_conic, cull_opacity) is packed into workspace_a, which
 *     must stay untouched until phase B has been enqueued.
 * b200gs_bin_sort: phase B (reads workspace_a only; cull = whether phase A was given the cull arrays).  Writes sorted_ids (Gaussian ids, front to back inside each tile; capacity max_pairs),
 *     tile_ranges[n_tiles,2] (int32 [start,end), clamped to max_pairs) and counts[2].  Coarse pairs beyond max_coarse
 *     and ids beyond max_pairs are DROPPED (never written out of bounds): the caller compares the counters with the
 *     capacities and redoes the phase with larger buffers if either overflowed.  max_pairs = counts[0] and
 *     max_coarse = counts[1] can never overflow. */
B200GS_API size_t b200gs_bin_count_workspace_bytes(int64_t n);
B200GS_API size_t b200gs_bin_sort_workspace_bytes(int64_t n, int64_t max_coarse, int32_t width, int32_t height);
B200GS_API int b200gs_bin_count(int32_t mode, int32_t width, int32_t height, int64_t n, const float* xy, const float* depth,
                     const int32_t* radii, const float* cull_conic, const float* cull_opacity, void* workspace_a, size_t workspace_a_bytes,
                     int64_t* d_counts, int64_t* host_counts, int32_t sync_host, void* stream);
B200GS_API int b200gs_bin_sort(int32_t mode, int32_t width, int32_t height, int64_t n, int32_t cull, int64_t max_coarse, int64_t max_pairs,
                    int64_t* d_counts, const void* workspace_a, void* workspace_b, size_t workspace_b_bytes, int32_t* sorted_ids,
                    int32_t* tile_ranges, int64_t* host_counts, int32_t sync_host, void* stream);

/* ---- gsplat intersection keys and tile offsets of one camera (C = 1) ---------------------------------------------------
 * The gsplat-v1 contract isect_tiles -> isect_offset_encode -> rasterize_to_pixels (gsplat_v1_renderer.py:446,458,500-520,588).
 * b200gs_isect_keys: gsplat's isect_ids of a binning, one per listed pair and in list order:
 *     keys[i] = (int64(tile) << 32) | float_bits(depth[sorted_ids[i]])      (camera bits 0)
 *     tile_ranges[n_tiles,2] / sorted_ids are b200gs_bin_sort's outputs with n_pairs = counts[2]; no range may end past n_pairs.
 *     The binning order is a stable sort of these keys, so they are non-decreasing and, without culling, equal to gsplat's
 *     sorted keys element for element.  A separate pass: the binning never builds them.
 *     Algorithmic bytes: 4 B id + 4 B depth gather (L2) in, 8 B key out per pair; 8 B range per tile.
 * b200gs_isect_offsets: gsplat's isect_offset_encode for C = 1: offsets[t] = index of the first of the n_pairs sorted keys whose
 *     tile (key >> 32) is >= t, for t < n_tiles (an empty tile gets the next non-empty start, tiles past the last key n_pairs;
 *     all 0 when n_pairs = 0).  Computed from the keys alone, by a binary search per tile: O(n_tiles log n_pairs) reads.
 *     n_pairs < 2^31. */
B200GS_API int b200gs_isect_keys(int32_t n_tiles, const int32_t* tile_ranges, const int32_t* sorted_ids, int64_t n_pairs, const float* depth,
                                 int64_t* keys, void* stream);
B200GS_API int b200gs_isect_offsets(int64_t n_pairs, const int64_t* keys, int32_t n_tiles, int32_t* offsets, void* stream);

/* b200gs_publish_i64: deliver n device int64 counters to host memory in stream order, the way the binning phases do
 *     (kernel with system-scope stores for pinned/mapped memory, cudaMemcpyAsync for pageable): for callers that run their
 *     own sync-free capacity protocol (the sharded renderer's row exchange). */
B200GS_API int b200gs_publish_i64(const int64_t* d_values, int64_t* host_values, int32_t n, void* stream);

/* ---- K6: blend forward ---------------------------------------------------------------------------------------------
 * replaces dgr renderCUDA fwd / gsplat rasterize_to_pixels fwd.  channels in {1,2,3,4}.
 * in : xy[n,2] conic[n,3] opacity[n] colors[n,channels]; bg[channels] or NULL.
 * out: image, addressed as image[pixel*pix_stride + channel*ch_stride] (vanilla [C,H,W]: pix_stride 1, ch_stride H*W;
 *      gsplat [H,W,C]: pix_stride C, ch_stride 1); final_T[H*W]; n_contrib[H*W] (1-based position in the tile's list of
 *      the last contributing splat); alpha[H*W] = 1 - final_T (nullable); hit_any[n] (nullable; caller zero-fills): 1 for every
 *      splat that contributed to at least one pixel, gsplat's `means2d.has_hit_any_pixels` (optimizers.py:39 SelectiveAdam;
 *      gsplat_v1_renderer.py:287 acc_vis). */
B200GS_API int b200gs_blend_fwd(int32_t mode, int32_t width, int32_t height, int32_t channels, const int32_t* tile_ranges,
                     const int32_t* sorted_ids, const float* xy, const float* conic, const float* opacity,
                     const float* colors, const float* bg, float* image, int64_t pix_stride, int64_t ch_stride,
                     float* final_T, int32_t* n_contrib, float* alpha, uint8_t* hit_any, void* stream);

/* ---- K7: blend backward --------------------------------------------------------------------------------------------
 * replaces dgr renderCUDA bwd / gsplat rasterize_to_pixels bwd.
 * in : forward inputs + final_T, n_contrib + v_image (same addressing as image) + v_alpha[H*W] (nullable).
 * out (ACCUMULATED with atomics — caller zero-fills): v_xy[n,2] (pixel units x (xy_scale_x, xy_scale_y)),
 *      v_conic[n,3], v_opacity[n], v_colors[n,channels]; v_xy_abs[n,2] (nullable; sum of |pixel grad|, gsplat absgrad). */
B200GS_API int b200gs_blend_bwd(int32_t mode, int32_t width, int32_t height, int32_t channels, const int32_t* tile_ranges,
                     const int32_t* sorted_ids, const float* xy, const float* conic, const float* opacity,
                     const float* colors, const float* bg, const float* final_T, const int32_t* n_contrib,
                     const float* v_image, int64_t pix_stride, int64_t ch_stride, const float* v_alpha,
                     float xy_scale_x, float xy_scale_y, float* v_xy, float* v_conic, float* v_opacity,
                     float* v_colors, float* v_xy_abs, void* stream);

/* ---- wide feature maps: K6 / K7 for any channel count (gsplat mode) ------------------------------------------------------
 * gsplat rasterize_gaussians with colors [n, D], D >= 1 — the reference's feature renderers composite 32-channel features
 * (internal/segany_splatting.py, seganygs_renderer.py, feature_3dgs_renderer.py).  Processed in chunks of 32 channels over the same
 * tile lists; per channel the arithmetic is K6's, so the composite of every channel is bit-identical to K6 on the same lists.
 * The background is added as one FMA, fmaf(final_T, bg[c], composite); K6 rounds final_T * bg[c] separately for some channels,
 * so with a background a channel may differ from K6's by that one rounding.
 * in : xy[n,2] conic[n,3] opacity[n] features[n,channels] (contiguous); bg[channels] or NULL.
 * fwd out: image[H,W,channels], final_T[H*W], n_contrib[H*W], alpha[H*W] = 1 - final_T (nullable).
 * bwd in : final_T, n_contrib, v_image[H,W,channels], v_alpha[H*W] (nullable).
 * bwd out (ACCUMULATED with atomics — caller zero-fills): v_features[n,channels]; v_xy[n,2] (pixel units), v_conic[n,3],
 *      v_opacity[n] — all three given, or all NULL for the features-only kernel (no geometry work at all); v_xy_abs[n,2]
 *      (nullable, needs v_xy): gsplat absgrad, exact for channels <= 32, the sum of each 32-channel chunk's value beyond. */
B200GS_API int b200gs_blend_feat_fwd(int32_t width, int32_t height, int32_t channels, const int32_t* tile_ranges, const int32_t* sorted_ids,
                                     const float* xy, const float* conic, const float* opacity, const float* features, const float* bg,
                                     float* image, float* final_T, int32_t* n_contrib, float* alpha, void* stream);
B200GS_API int b200gs_blend_feat_bwd(int32_t width, int32_t height, int32_t channels, const int32_t* tile_ranges, const int32_t* sorted_ids,
                                     const float* xy, const float* conic, const float* opacity, const float* features, const float* bg,
                                     const float* final_T, const int32_t* n_contrib, const float* v_image, const float* v_alpha,
                                     float* v_features, float* v_xy, float* v_conic, float* v_opacity, float* v_xy_abs, void* stream);

/* ---- fused L1 + SSIM training loss on the rendered image (validated by tests/test_gpu_loss.py) ----------------------------------
 * replaces  loss = (1-lambda) * l1_loss(image, gt) + lambda * (1 - ssim(image, gt))   (internal/metrics/vanilla_metrics.py:57-74,
 * internal/utils/ssim.py:17-63: 11-tap Gaussian window sigma 1.5, zero padding, C1 = 0.01^2, C2 = 0.03^2).  image/target [C,H,W].
 * b200gs_loss_fwd: partials[b200gs_loss_blocks(...)][2] <- per-CTA sums of |image-target| and of the SSIM map (the caller sums them
 *     and divides by C*H*W); dmaps[3][C][H][W] <- partial derivatives of the SSIM map, kept for the backward.
 * b200gs_loss_bwd: v_image[C,H,W] <- (*v_loss or 1) * dloss/dimage.
 * Sizes: 1 <= channels <= 65535, 1 <= height <= 65535 * 16 and 1 <= width <= 2^31 - 16 (the launch grid is ceil(W/16) x ceil(H/16)
 * x C); fwd and bwd return B200GS_EINVAL for other sizes or a NULL pointer (v_loss may be NULL) before any CUDA call, and
 * b200gs_loss_blocks returns 0 for them. */
B200GS_API int64_t b200gs_loss_blocks(int32_t channels, int32_t width, int32_t height);
B200GS_API int b200gs_loss_fwd(int32_t channels, int32_t width, int32_t height, const float* image, const float* target, float* dmaps,
                               float* partials, void* stream);
B200GS_API int b200gs_loss_bwd(int32_t channels, int32_t width, int32_t height, const float* image, const float* target, const float* dmaps,
                               float lambda_dssim, const float* v_loss, float* v_image, void* stream);

/* ---- [n,12] splat rows: the exchange format of the Gaussian-sharded multi-GPU renderer ------------------------------
 * replaces the packing / splitting around the reference's all-to-all of projected splats
 * (internal/renderers/gsplat_distributed_renderer.py:127-217): one fp32 row per VISIBLE Gaussian,
 *   col 0-1 xy | 2 depth | 3-5 conic | 6 compensation | 7 opacity | 8-10 rgb | 11 radius (int32 bit pattern).
 * b200gs_pack_rows: compacts the visible (radii > 0) entries of K1's outputs into rows, in index order; row_index[n] (int32)
 *     = the row of entry i, kept for the backward; *d_count <- number of rows.
 * b200gs_bin_count_rows (then b200gs_bin_sort) / blend_fwd_rows / blend_bwd_rows: K2-K7 reading the rows IN PLACE (strided
 *     access, no split copies); blend_bwd_rows accumulates into a zero-filled [n,12] gradient row buffer that goes
 *     straight back through the all-to-all.  3 colour channels; cull != 0 enables exact tile culling.
 *     blend_fwd_rows / blend_bwd_rows read rows (and blend_bwd_rows accumulates into v_rows) with 16-byte accesses: both buffers
 *     must be 16-byte aligned (an allocation base is), or the call fails with B200GS_EINVAL. */
#define B200GS_MAX_VIEWS 8      /* cameras per multi-view launch / destination ranks per peer-mode pack (one NVSwitch box) */
/* b200gs_project_pack_multi numbers camera j's rows j*block_rows + k in an int32 row_index: it requires
 * n_views * block_rows <= 2^31 - 1 (with B200GS_MAX_VIEWS views, block_rows <= 268435455) and returns B200GS_EINVAL otherwise. */
#define B200GS_ROW_FLOATS 12
#define B200GS_ROW_XY 0
#define B200GS_ROW_DEPTH 2
#define B200GS_ROW_CONIC 3
#define B200GS_ROW_COMP 6
#define B200GS_ROW_OPACITY 7
#define B200GS_ROW_RGB 8
#define B200GS_ROW_RADIUS 11
/* Fused activations ("raw parameters"): the K1 / K8 entry points below read the RAW parameter tensors of VanillaGaussianModel
 *     (internal/models/vanilla_gaussian.py:66,345-358; internal/models/gaussian.py:250-254) instead of its getters: scales =
 *     exp(log_scales), quats = normalize(raw_quats), opacity = sigmoid(opacity_logits) (all evaluated inside the kernel, the geometry
 *     part in fp64), SH = shs_dc[n,1,3] | shs_rest[n,sh_stride-1,3] read in place (no torch.cat).  The blend opacity is that opacity
 *     x compensation in gsplat mode when anti_aliased != 0 (gsplat_renderer.py:81-83); gradients are w.r.t. the RAW tensors.
 * b200gs_project_fwd_rows: K1 (fused activations, either constant set) writing ONE [n,12] row per Gaussian instead of the separate
 *     arrays — the single-GPU renderers' fast path: K2-K7 read the rows in place (b200gs_bin_count_rows, b200gs_blend_fwd_rows,
 *     b200gs_blend_bwd_rows), K8 reads the gradient rows (b200gs_project_bwd_rows with row_offsets = NULL).  Rows of culled
 *     Gaussians have radius 0, zeros in columns 0..3 and 8..10 (columns 4..7 unspecified).  radii[n], clamped[n] (what K8 needs) are written too; tiles may be NULL. */
B200GS_API int b200gs_project_fwd_rows(const B200gsView* view, int64_t n, const float* means, const float* log_scales,
                                       const float* raw_quats, const float* opacity_logits, const float* shs_dc, const float* shs_rest,
                                       int32_t anti_aliased, float* rows, int32_t* radii, uint8_t* clamped, int32_t* tiles, void* stream);
/* b200gs_project_bwd_rows: K8 (fused activations) taking its cotangents straight from compacted [V,12] gradient rows
 *     (v_rows[row_offsets[i]] for visible i; row_offsets = NULL: v_rows[i]) and, when accumulate != 0, ADDING to the gradient buffers — the sharded
 *     renderer calls it once per camera of the step without unpack copies or separate sum kernels.
 *     v_mean2d (optional, may be NULL): [n, v_mean2d_cols] (2 or 3 columns) <- dL/dmean2D of every Gaussian (columns 0..1 of its gradient row; zeros
 *     for culled Gaussians and in column 2): the `.grad` of the renderer contract's `viewspace_points` (vanilla_renderer.py:55-56,
 *     vanilla_density_controller.py:101-123), written here instead of by a fill + strided copy after the kernel. */
B200GS_API int b200gs_project_bwd_rows(const B200gsView* view, int64_t n, const float* means, const float* log_scales,
                                       const float* raw_quats, const float* opacity_logits, const float* shs_dc, const float* shs_rest,
                                       int32_t anti_aliased, const int32_t* radii, const uint8_t* clamped, const int32_t* row_offsets,
                                       const float* v_rows, int32_t accumulate, float* v_means, float* v_log_scales, float* v_raw_quats,
                                       float* v_opacity_logits, float* v_shs_dc, float* v_shs_rest, float* v_mean2d, int32_t v_mean2d_cols,
                                       void* stream);
/* b200gs_project_fwd_raw_multi / b200gs_project_bwd_rows_multi: K1 / K8 of one shard for ALL n_views (<= B200GS_MAX_VIEWS) cameras of a
 *     step in one launch each (gsplat constants, raw parameters; sh_degree / sh_stride / scale_modifier of views[0] apply to all).
 *     fwd: camera-major outputs, view j at elements [j*n, (j+1)*n); parameters and SH blocks are read once per Gaussian.
 *     bwd: every thread accumulates its Gaussian's gradients over the cameras in registers and writes them once; cotangents are
 *     [.,12] gradient rows, entry (j, i) reads row row_index[j*n+i] of v_rows[j] — a HOST array of n_views device pointers, each
 *     of which may address a peer GPU's buffer (the camera owner's gradient rows are pulled over NVLink, no return all-to-all). */
B200GS_API int b200gs_project_fwd_raw_multi(const B200gsView* views, int32_t n_views, int64_t n, const float* means, const float* log_scales,
                                            const float* raw_quats, const float* opacity_logits, const float* shs_dc, const float* shs_rest,
                                            int32_t anti_aliased, float* xy, float* depth, int32_t* radii, float* conic, float* rgb,
                                            uint8_t* clamped, float* opacity_out, void* stream);
/* b200gs_project_pack_multi: K1 of one shard for all n_views cameras FUSED with the packing of the exchange.  The visible splats of
 *     camera j leave the kernel as [.,12] rows, in Gaussian-index order, stored straight into dst_rows[j] (a HOST array of n_views device
 *     pointers: block of block_rows rows in the receive buffer of the rank that owns camera j — peer memory over NVLink — or in a local
 *     send buffer); rows past block_rows are dropped.  d_count[j] = visible splats of camera j (compare with block_rows).  Kept locally
 *     for K8 and the renderer contract, camera-major ([j*n + i]): xy (mean2D), radii, clamped, row_index (j*block_rows + k, -1 = dropped).
 *     Sizes: 1 <= n_views <= B200GS_MAX_VIEWS, 0 <= n < 2^30, 1 <= block_rows < 2^30, n_views * block_rows <= 2^31 - 1, dst_rows[j]
 *     16-byte aligned, workspace_bytes >= b200gs_project_pack_workspace_bytes when n > 0; B200GS_EINVAL otherwise, before any CUDA call.
 *     Replaces b200gs_project_fwd_raw_multi + b200gs_pack_rows (gsplat_distributed_renderer.py:127-217: project, then all-to-all). */
B200GS_API size_t b200gs_project_pack_workspace_bytes(int32_t n_views, int64_t n);
B200GS_API int b200gs_project_pack_multi(const B200gsView* views, int32_t n_views, int64_t n, const float* means, const float* log_scales,
                                         const float* raw_quats, const float* opacity_logits, const float* shs_dc, const float* shs_rest,
                                         int32_t anti_aliased, float* xy, int32_t* radii, uint8_t* clamped, int32_t* row_index,
                                         void* const* dst_rows, int64_t block_rows, void* workspace, size_t workspace_bytes,
                                         int64_t* d_count, void* stream);
B200GS_API int b200gs_project_bwd_rows_multi(const B200gsView* views, int32_t n_views, int64_t n, const float* means, const float* log_scales,
                                             const float* raw_quats, const float* opacity_logits, const float* shs_dc, const float* shs_rest,
                                             int32_t anti_aliased, const int32_t* radii, const uint8_t* clamped, const int32_t* row_index,
                                             const float* const* v_rows, float* v_means, float* v_log_scales, float* v_raw_quats,
                                             float* v_opacity_logits, float* v_shs_dc, float* v_shs_rest, void* stream);
/* b200gs_ipc_alloc / _handle / _open / _close / _free: device buffers that peer processes of the same box can map (cudaMalloc +
 *     CUDA IPC): the exchange buffers of the sharded renderer.  handle = 64 bytes to pass to the peers by any host channel. */
B200GS_API int b200gs_ipc_alloc(size_t bytes, void** dev_ptr, unsigned char* handle64);
B200GS_API int b200gs_ipc_open(const unsigned char* handle64, void** dev_ptr);
B200GS_API int b200gs_ipc_close(void* dev_ptr);
B200GS_API int b200gs_ipc_free(void* dev_ptr);
B200GS_API size_t b200gs_pack_rows_workspace_bytes(int64_t n);
B200GS_API int b200gs_pack_rows(int64_t n, const float* xy, const float* depth, const float* conic, const float* comp, const float* opacity,
                                const float* rgb, const int32_t* radii, void* workspace, size_t workspace_bytes, int32_t* row_index,
                                float* rows, int64_t* d_count, void* stream);
/* b200gs_bin_count_rows reads every row with three 16-byte loads: rows must be 16-byte aligned (an allocation base is), or the call
 *     fails with B200GS_EINVAL.  It always packs the conic and opacity columns for phase B, so its cull argument has no effect: the cull
 *     argument of b200gs_bin_sort decides whether the tiles are culled.
 * block_counts / block_rows (optional; NULL / 0 = every row counts): the rows arrive in blocks of block_rows rows of which only the first
 *     block_counts[b] are valid (the fixed-capacity exchange of the sharded renderer) — the rest reads as culled, so the receive buffer
 *     needs no padding pass.  With block_counts, block_rows must be 1..2^31 - 1 (B200GS_EINVAL otherwise). */
B200GS_API int b200gs_bin_count_rows(int32_t mode, int32_t width, int32_t height, int64_t n, const float* rows, int32_t cull,
                                     void* workspace_a, size_t workspace_a_bytes, int64_t* d_counts, int64_t* host_counts,
                                     int32_t sync_host, void* stream, const int64_t* block_counts, int64_t block_rows);
B200GS_API int b200gs_blend_fwd_rows(int32_t mode, int32_t width, int32_t height, const int32_t* tile_ranges, const int32_t* sorted_ids,
                                     const float* rows, const float* bg, float* image, int64_t pix_stride, int64_t ch_stride,
                                     float* final_T, int32_t* n_contrib, float* alpha, void* stream);
/* grad_scale_x / _y: factor on the mean2D columns of the gradient rows (vanilla renderers: 0.5 W, 0.5 H — the vanilla rasterizer's
 *     NDC-unit convention; gsplat renderers: 1, 1).  v_rows must be zero-filled: the kernel accumulates with 128-bit reductions. */
B200GS_API int b200gs_blend_bwd_rows(int32_t mode, int32_t width, int32_t height, const int32_t* tile_ranges, const int32_t* sorted_ids,
                                     const float* rows, const float* bg, const float* final_T, const int32_t* n_contrib,
                                     const float* v_image, int64_t pix_stride, int64_t ch_stride, const float* v_alpha,
                                     float grad_scale_x, float grad_scale_y, float* v_rows, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200GS_H */
