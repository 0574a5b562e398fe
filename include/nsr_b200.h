/* nsr_b200 -- C ABI of the H100 (sm_90a) per-ray rendering hot path (drop-in for the tiny-cuda-nn +
 * nerfacc 0.3.3 calls made by bennyguo/instant-nsr-pl's models/).
 *
 * Conventions (SURVEY.md §8b):
 *  - plain pointers + sizes, no torch types.  Every pointer is a DEVICE pointer unless it says host.
 *  - the caller owns all memory (inputs, outputs, workspace); the library never allocates or frees
 *    device memory and keeps no pointer after return.
 *  - every entry point takes the CUDA stream explicitly (void* = cudaStream_t), is re-entrant and
 *    thread-safe (forward runs on the main Python thread, backward on autograd's worker thread).
 *  - return 0 on success; non-zero => message in nsr_last_error() (thread-local).
 *  - variable-length outputs use count -> (caller allocates) -> write, or device-side counts with
 *    caller-provided capacity.
 *
 * Each declaration cites the reference interface it replaces (paths relative to the reference repo).
 */
#ifndef NSR_B200_H
#define NSR_B200_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NSR_MAX_LEVELS 32
#define NSR_VERSION 100

/* Hash-grid geometry.  Replaces the encoding_config dict handed to tcnn.Encoding /
 * tcnn.NetworkWithInputEncoding (models/network_utils.py:47,90,209; configs/nerf-blender.yaml:43-49).
 * The per-level table is computed once on the host (fp32, identical to oracle/hashgrid.py). */
typedef struct {
  int32_t n_levels;
  int32_t n_features;              /* per level; only 2 is implemented (every reference config) */
  float scale[NSR_MAX_LEVELS];     /* exp2(l*log2(pls))*base - 1 */
  uint32_t res[NSR_MAX_LEVELS];    /* ceil(scale)+1 */
  uint32_t size[NSR_MAX_LEVELS];   /* entries in level */
  uint32_t offset[NSR_MAX_LEVELS]; /* first entry of level */
  uint32_t dense_mask;             /* bit l set: dense indexing, else coherent-prime hash */
} nsr_grid_t;

/* Fully-fused MLP description.  Replaces network_config of tcnn.Network (models/network_utils.py:181;
 * configs/nerf-blender.yaml:50-55,62-67).  Width is fixed at 64 (every reference config). */
typedef struct {
  int32_t n_in;        /* logical input width; padded to a multiple of 16 with ones */
  int32_t n_out;       /* logical output width (<= 16) */
  int32_t n_hidden;    /* number of hidden layers (1..3) */
  int32_t activation;  /* hidden: 0 none, 1 relu */
  int32_t out_activation; /* 0 none, 1 relu, 2 sigmoid, 3 exponential */
} nsr_mlp_t;

/* Occupancy grid + marching parameters.  Replaces nerfacc.OccupancyGrid state and the kwargs of
 * nerfacc.ray_marching (models/nerf.py:36-41,82-93; models/neus.py:63-74,159-169,210-220). */
typedef struct {
  float roi[6];            /* roi_aabb */
  int32_t res;             /* grid resolution per axis */
  int32_t contraction;     /* 0 AABB, 2 UN_BOUNDED_SPHERE (nerfacc.ContractionType) */
  float step;              /* render_step_size */
  float cone_angle;
} nsr_march_t;

/* Fused NeRF field of the nerf-blender shape (configs/nerf-blender.yaml:30-67): HashGrid(L=16,F=2) ->
 * FullyFused 32->64->feature_dim(16), density = trunc_exp(out0 + density_bias); colour = sigmoid(FullyFused
 * [feature(16) | SH4(dir)(16)] -> 64 -> 64 -> 3); AABB contraction x01 = (x + radius) / (2 radius).
 * Replaces VolumeDensity.forward + VolumeRadiance.forward (models/geometry.py:122-130, models/texture.py:23-30). */
typedef struct {
  nsr_grid_t grid;
  float radius;
  float density_bias;
  int32_t feature_dim;     /* must be 16 */
  int32_t density_hidden;  /* must be 1 */
  int32_t color_hidden;    /* must be 2 */
  int32_t contraction;     /* 0 AABB (above), 2 UN_BOUNDED_SPHERE: x01 -> v = 2 x01 - 1, |v| > 1 -> (2 - 1/|v|) v/|v|, then v/4 + 1/2
                              (models/geometry.py contract_to_unisphere); honoured by nsr_nerf_density / _prepass / _render_fwd /
                              nsr_nerf_field_bwd without xyzdir; every other entry point needs 0 */
} nsr_nerf_t;

/* VolumeRadiance fused kernel (models/texture.py:23-30): input = cat[feature (n_feat) | SH degree 4 of the ray direction (16) |
 * extra (n_extra, NeuS: the unit normal)], which must be 32 wide; FullyFused 64-wide MLP with two hidden ReLU layers, 3 outputs.
 * act_mode 0: raw network output; 1: Sigmoid as the network's output activation (nerf-blender.yaml:66, result rounded to fp16);
 * 2: no network activation, fp32 sigmoid afterwards (neus-blender.yaml `color_activation: sigmoid`). */
typedef struct {
  int32_t n_feat;
  int32_t n_extra;
  int32_t act_mode;
} nsr_radiance_t;

/* torch.optim.AdamW hyper-parameters (systems/utils.py:314-325; nerf-blender.yaml:74-79: lr 1e-2, betas (0.9, 0.99), eps 1e-15,
 * weight_decay = torch's default 1e-2).  step: 1-based number of THIS update; inv_grad_scale: gradients are multiplied by it
 * first (1 / GradScaler scale; 1 for none). */
typedef struct {
  float lr, beta1, beta2, eps, weight_decay;
  int32_t step;
  float inv_grad_scale;
} nsr_adamw_t;

/* weights of the NeuS training losses (systems/neus.py:98-121; configs/neus-blender.yaml:80-89) */
typedef struct {
  float lambda_rgb_mse, lambda_rgb_l1, lambda_eikonal, lambda_mask, lambda_opaque, lambda_sparsity, sparsity_scale;
} nsr_neus_loss_t;



const char* nsr_last_error(void);
int nsr_version(void);
int nsr_device_info(int* sm_count, int* cc_major, int* cc_minor);

/* ---- encodings / networks (tiny-cuda-nn surface) -------------------------------------------- */

/* tcnn.Encoding(HashGrid).forward  (models/network_utils.py:47,90).  x [n,3] f32 in [0,1];
 * table fp16 [entries,2]; out fp16 [n, L*2]. */
int nsr_hashgrid_fwd(const nsr_grid_t* g, const float* x, const void* table_h, void* out_h, int64_t n, void* stream);
/* autograd of the above w.r.t. the table: grad_table f32 [entries*2] += dy_scale * scatter (atomic, one
 * 8-byte vector RED per corner). dy fp16 [n,L*2] (possibly loss-scaled; dy_scale undoes it in fp32). */
int nsr_hashgrid_bwd(const nsr_grid_t* g, const float* x, const void* dy_h, float* grad_table, float dy_scale, int64_t n, void* stream);
/* ... w.r.t. the input (NeuS analytic normals, models/geometry.py:177-180): dx f32 [n,3]. dy f32 [n,L*2]. */
int nsr_hashgrid_bwd_input(const nsr_grid_t* g, const float* x, const void* table_h, const float* dy, float* dx, int64_t n, void* stream);
/* double backward of bwd_input (eikonal loss, systems/neus.py:106-108): given ddx f32 [n,3]
 * -> grad_table += d/dtable, grad_dy f32 [n,L*2] (either may be NULL). */
int nsr_hashgrid_bwd_bwd(const nsr_grid_t* g, const float* x, const void* table_h, const float* dy, const float* ddx,
                         float* grad_table, float* grad_dy, int64_t n, void* stream);

/* tcnn.Encoding(SphericalHarmonics, degree 4).forward (models/network_utils.py:90; texture.py:24-25).
 * v [n,3] f32 in [0,1]; out fp16 [n,16]. */
int nsr_sh4_fwd(const float* v, void* out_h, int64_t n, void* stream);

/* tcnn.Network(FullyFusedMLP).forward (models/network_utils.py:181).  x fp16 [n, in_pad]; params fp16
 * flat (row-major [out,in] matrices, tcnn layout); out fp16 [n,16]. */
int nsr_mlp_fwd(const nsr_mlp_t* m, const void* x_h, const void* params_h, void* out_h, int64_t n, void* stream);
/* autograd of the above: dy fp16 [n,16] (w.r.t. post-activation output).  dy is multiplied by loss_scale
 * on load (tcnn uses 128) so the fp16 dgrad chain stays in range; grad_params f32 flat += TRUE gradient;
 * dx fp16 [n,in_pad] (may be NULL) = loss_scale * true gradient. */
int nsr_mlp_bwd(const nsr_mlp_t* m, const void* x_h, const void* params_h, const void* y_h, const void* dy_h,
                float* grad_params, void* dx_h, float loss_scale, int64_t n, void* stream);
/* The reference's VanillaMLP with ReLU (models/network_utils.py:95-139: nn.Linear WITH biases, fp32 in/out under autocast(False))
 * on the same kernels: x fp16 [n, in_pad] (columns beyond n_in zero), weights_h fp16 in the FullyFused layout above (W1 columns
 * beyond n_in zero, last matrix rows beyond n_out zero), bias f32 [64 * n_hidden + 16], out f32 [n, n_out] (compact).  fp16
 * tensor-core operands, fp32 accumulation starting from the bias.  Backward: dy f32 [n, n_out]; grad_weights f32 (+=, layout of
 * weights_h), grad_bias f32 [64 * n_hidden + 16] (+=), dx f32 [n, n_in] = dL/dx (compact, unscaled; may be NULL); loss_scale > 0
 * fixes the scale of the fp16 dgrad chain, <= 0 derives it from *amax (device float: max |dy|). */
int nsr_mlp_vanilla_fwd(const nsr_mlp_t* m, const void* x_h, const void* weights_h, const float* bias, float* out, int64_t n,
                        void* stream);
int nsr_mlp_vanilla_bwd(const nsr_mlp_t* m, const void* x_h, const void* weights_h, const float* bias, const float* dy,
                        float* grad_weights, float* grad_bias, float* dx, float loss_scale, const float* amax, int64_t n, void* stream);

/* Warpgroup-MMA (wgmma) version of nsr_mlp_fwd (same tensors): 128-row CTA tiles, operands in the canonical K-major smem layout,
 * fp32 accumulators in registers.  variant bit 0 = swap LBO/SBO in the smem descriptors (a layout check: wrong results);
 * status: accepted for ABI compatibility, never written. */
int nsr_mlp_fwd_tc(const nsr_mlp_t* m, const void* x_h, const void* params_h, void* out_h, int64_t n, int variant, int* status, void* stream);

/* ---- marching / compositing (nerfacc 0.3.3 surface) ----------------------------------------- */

/* nerfacc.intersection.ray_aabb_intersect (models/neus.py:153). */
int nsr_ray_aabb(const float* rays_o, const float* rays_d, const float* aabb6, float* t_min, float* t_max, int64_t n, void* stream);
/* nerfacc.ray_marching, pass 1: per-ray sample counts (models/nerf.py:83).  t_min/t_max are the
 * prepared per-ray intervals; bits = packed occupancy (bit idx&31 of word idx>>5). */
int nsr_march_count(const nsr_march_t* p, const float* rays_o, const float* rays_d, const float* t_min, const float* t_max,
                    const uint32_t* bits, int32_t* counts, int64_t n_rays, void* stream);
/* exclusive scan of counts -> offsets[n+1] (offsets[n] = total). */
int nsr_scan_counts(const int32_t* counts, int64_t* offsets, int64_t n, void* stream);
/* pass 2: write samples at offsets. */
int nsr_march_write(const nsr_march_t* p, const float* rays_o, const float* rays_d, const float* t_min, const float* t_max,
                    const uint32_t* bits, const int64_t* offsets, int32_t* ray_indices, float* t_starts, float* t_ends,
                    int64_t n_rays, void* stream);

/* nerfacc render_visibility (inside ray_marching, models/nerf.py:87-92): per ray, exclusive
 * transmittance from alpha; keep[i] = T_i >= eps && (alpha_thre<=0 || alpha>=thre). */
int nsr_visibility(const float* alphas, const int64_t* offsets, uint8_t* keep, float* trans, int32_t* kept_counts,
                   float early_stop_eps, float alpha_thre, int64_t n_rays, void* stream);
/* nerfacc.render_weight_from_density / _from_alpha fwd+bwd (models/nerf.py:105, neus.py:237).
 * `trans` (exclusive transmittance T_i, may be NULL in fwd) is what the backward needs:
 *   d sigma_i = delta_i [ g_i (T_i - w_i) - sum_{j>i} g_j w_j ],  d alpha_i = g_i T_i - sum_{j>i} g_j w_j / (1 - alpha_i). */
int nsr_weight_from_density_fwd(const float* t_starts, const float* t_ends, const float* sigmas, const int64_t* offsets,
                                float* weights, float* trans, int64_t n_rays, void* stream);
int nsr_weight_from_density_bwd(const float* t_starts, const float* t_ends, const float* weights, const float* trans,
                                const float* grad_weights, const int64_t* offsets, float* grad_sigmas, int64_t n_rays, void* stream);
int nsr_weight_from_alpha_fwd(const float* alphas, const int64_t* offsets, float* weights, float* trans, int64_t n_rays, void* stream);
int nsr_weight_from_alpha_bwd(const float* alphas, const float* weights, const float* trans, const float* grad_weights,
                              const int64_t* offsets, float* grad_alphas, int64_t n_rays, void* stream);
/* nerfacc.accumulate_along_rays (models/nerf.py:106-108): out[n_rays,d] = segmented sum of w*v. */
int nsr_accumulate(const float* weights, const float* values, const int64_t* offsets, float* out, int32_t d, int64_t n_rays, void* stream);

/* ---- fused NeRF path (module-level surface: NeRFModel.forward_, models/nerf.py:61-127) ----------------
 * Sample counts may live on the device: where an entry point takes (n, n_dev), a non-NULL n_dev (device int64)
 * holds the true count and n is the buffer capacity -- no host sync, so a whole step can be captured in a CUDA
 * graph.  n_dev == NULL: n is the count. */

/* marching for the fused path (AABB, cone_angle 0; same sample sets as nsr_ray_aabb + nsr_march_count/_write):
 * one kernel does ray-box intersection (+ per-ray jitter * step when jitter != NULL), tests the step lattice
 * against the bitfield (coarse_bits: optional (res/4)^3 "any bit in the 4^3 block" field used to skip empty space),
 * stores the per-ray occupancy masks [n_rays, words], t_min and the per-ray sample counts.
 * nsr_scan_counts_order: exclusive scan of the counts + a longest-rays-first processing order (rays bucketed by their
 * number of 32-sample chunks) for the per-ray kernel.  nsr_march_rays_expand turns the masks into packed samples. */
/* nsr_march_rays_alloc: nsr_march_rays_mask + slice allocation + queue binning in the same launch (replaces nsr_scan_counts_order).
 * Reference call site: nerfacc.ray_marching in NeRFModel.forward_ (models/nerf.py:82-93) -- what nerfacc does with a host-synchronised exact
 * allocation (`num_steps.sum().item()`), done on the device:
 *   offsets[ray] = atomic reservation of counts[ray] rows (completion order, not ray order; *alloc_total (uint64, zero on entry) ends as the
 *   number of marched samples); bin_counts int32[8] (zero on entry) / order_bins int32[8 * n]: rays grouped by 32-sample chunk count
 *   (>= 17, 13-16, 9-12, 5-8, 3-4, 2, 1, 0), the queue of nsr_nerf_rays_fwd (pass counts + bin_counts there). */
int nsr_march_rays_alloc(const nsr_march_t* p, const float* rays, const float* jitter, const uint32_t* bits, const uint32_t* coarse_bits,
                         uint32_t* masks, int32_t words, float* t_min, int32_t* counts, int64_t* offsets, void* alloc_total,
                         int32_t* bin_counts, int32_t* order_bins, int64_t n, void* stream);
int nsr_march_rays_mask(const nsr_march_t* p, const float* rays, const float* jitter, const uint32_t* bits, const uint32_t* coarse_bits,
                        uint32_t* masks, int32_t words, float* t_min_out, int32_t* counts, int64_t n_rays, void* stream);
int nsr_scan_counts_order(const int32_t* counts, int64_t* offsets, int32_t* order, int64_t n, void* stream);
int nsr_march_rays_expand(const nsr_march_t* p, const uint32_t* masks, int32_t words, const float* t_min, const int64_t* offsets,
                          int32_t* ray_indices, float* t_starts, float* t_ends, int64_t n_rays, void* stream);
/* marching for the unbounded fused path (cone_angle > 0, any contraction; same sample sets as nsr_march_count/_write given the same
 * intervals): one warp per ray; every lane runs the same fp32 step recurrence t1 = t0 + min(max(t0 * cone, step), 1e10) for a 32-step
 * chunk and lane k tests step k against the bitfield.  Per-ray interval in nerfacc's order: t_min = max(t_min_in[ray] or 0, near),
 * t_max = min(t_max_in[ray] or 1e10, far), then t_min += jitter[ray] * step when jitter != NULL (t_min_in / t_max_in / jitter may be
 * NULL; pass near = -inf / far = +inf for none).  nsr_march_cone_mask writes per-ray masks [n_rays, words] (words * 32 = the step bound of
 * a ray: it never takes more steps), the per-ray counts and the ray's first t (t_start [n_rays]); nsr_scan_counts turns the counts into
 * ray-ordered offsets.  nsr_march_cone_expand recomputes the recurrence and writes packed samples at offsets; rows at or past cap are
 * not written, and a ray reaching past cap sets *overflow (device int32, may be NULL) to 1. */
int nsr_march_cone_mask(const nsr_march_t* p, const float* rays, const float* jitter, const float* t_min_in, const float* t_max_in, float near,
                        float far, const uint32_t* bits, uint32_t* masks, int32_t words, float* t_start, int32_t* counts, int64_t n_rays,
                        void* stream);
int nsr_march_cone_expand(const nsr_march_t* p, const uint32_t* masks, int32_t words, const float* t_start, const int64_t* offsets,
                          int32_t* ray_indices, float* t_starts, float* t_ends, int64_t cap, int32_t* overflow, int64_t n_rays, void* stream);
/* density at world positions (occ_eval_fn of models/nerf.py:49-52; VolumeDensity.forward density-only).
 * positions f32 [n,3]; dparams fp16 flat [3072 MLP | table]; density f32 [n]. */
int nsr_nerf_density(const nsr_nerf_t* f, const float* positions, const void* dparams_h, float* density, int64_t n, void* stream);
/* sigma_fn pre-pass of ray_marching (models/nerf.py:65-71,87): marched samples (ray_indices i32, t_starts,
 * t_ends [m]) over rays f32 [n_rays,6] -> alphas[m] = 1 - exp(-sigma * (t_end - t_start)). */
int nsr_nerf_prepass(const nsr_nerf_t* f, const float* rays, const int32_t* ray_indices, const float* t_starts, const float* t_ends,
                     const void* dparams_h, float* alphas, int64_t m, const int64_t* m_dev, void* stream);
/* boolean-mask compaction of the pre-pass (the three `tensor[mask]` of nerfacc.ray_marching): with alpha_thre == 0
 * the kept samples of a ray are a prefix, so ray r's first kept_counts[r] samples move from offsets_m[r] to
 * offsets_k[r].  trans (exclusive transmittance from nsr_visibility) travels with them. */
int nsr_compact_prefix(const int64_t* offsets_m, const int64_t* offsets_k, const int32_t* ray_indices_m, const float* t_starts_m,
                       const float* t_ends_m, const float* trans_m, int32_t* ray_indices_k, float* t_starts_k, float* t_ends_k,
                       float* trans_k, int64_t n_rays, void* stream);
/* main pass (models/nerf.py:95-108): kept samples -> per-sample sigma, rgb, weights (= trans * (1 - exp(-sigma delta)))
 * and per-ray sums acc_rgb[n_rays,3], opacity[n_rays], depth[n_rays] (must be zeroed by the caller; atomically
 * accumulated).  enc_save (fp16 [k,32], may be NULL) keeps the encoded features for the backward pass. */
int nsr_nerf_render_fwd(const nsr_nerf_t* f, const float* rays, const int32_t* ray_indices, const float* t_starts, const float* t_ends,
                        const float* trans, const void* dparams_h, const void* cparams_h, void* enc_save_h, float* sigmas, float* rgbs,
                        float* weights, float* acc_rgb, float* opacity, float* depth, int64_t k, const int64_t* k_dev, void* stream);
/* backward through the compositing (autograd of render_weight_from_density + accumulate_along_rays x3) and the
 * density activation: per-ray grads (g_rgb [n_rays,3], g_opacity, g_depth [n_rays]; g_weights [k] optional) ->
 * d_sraw [k] = dL/d(out0) (trunc_exp backward, models/utils.py:64-66, folded in), d_rgb [k,3].
 * amax (device float, zeroed by the caller, may be NULL) receives max(|d_sraw|, |d_rgb|/4) for loss scaling. */
int nsr_nerf_ray_bwd(const int64_t* offsets_k, const float* t_starts, const float* t_ends, const float* trans, const float* weights,
                     const float* sigmas, const float* rgbs, const float* g_rgb, const float* g_opacity, const float* g_depth,
                     const float* g_weights, float* d_sraw, float* d_rgb, float* amax, int64_t n_rays, void* stream);
/* backward through both networks and the hash grid (autograd of VolumeRadiance + VolumeDensity + HashGrid):
 * recomputes the forward from enc_save on tensor cores; grad_dparams f32 [3072 + table] and grad_cparams f32 [7168]
 * are accumulated atomically (caller zeroes).  loss_scale keeps the fp16 dgrad chain in range; <= 0 selects it
 * on the device from *amax (no host sync). */
int nsr_nerf_field_bwd(const nsr_nerf_t* f, const float* rays, const int32_t* ray_indices, const float* t_starts, const float* t_ends,
                       const void* enc_save_h, const void* dparams_h, const void* cparams_h, const float* d_sraw, const float* d_rgb,
                       float* grad_dparams, float* grad_cparams, float loss_scale, const float* amax, int64_t k, const int64_t* k_dev,
                       const int64_t* row_pos /* optional: row j of enc_save / d_sraw / d_rgb lives at row_pos[j] (loose layout) */,
                       const float* xyzdir /* optional f32 [k,6]: unit-cube position + view direction per row (nsr_pack_kept); then rays,
                                              ray_indices, t_starts, t_ends are not read and every load of a tile is independent */,
                       void* stream);
/* ---- the same two-pass field with the reference's VanillaMLP networks (NeuS learned background, configs/neus-dtu.yaml:72-105) ----
 * f: contraction = 2 (UN_BOUNDED_SPHERE) only; L=16 F=2 grid, feature_dim 16, hidden layers 1 / 2 as above.  The networks are nn.Linear
 * with fp32 biases, packed by the caller into the FullyFused layouts so that the kernels keep their shapes:
 *   dmlp_h fp16 [3072] = W1 [64][32] | W2 [16][64], rows 8..15 of W2 zero;  dbias f32 [80] = b1 [64] | b2 [16], entries 8..15 zero
 *     (feature_dim 8: feature columns 8..15 are exactly 0);
 *   cmlp_h fp16 [7168] = W1 [64][32] | W2 [64][64] | W3 [16][64], W1 = [W[:, 0:8] | 0 (8 columns) | W[:, 8:24]] of the [64][24] layer
 *     (features in input columns 0..15, SH4 in 16..31), rows 3..15 of W3 zero;  cbias f32 [144] = b1 [64] | b2 [64] | b3 [16].
 *   table_h fp16: the hash table, its own buffer (not behind the density network as in nsr_nerf_*).
 * Rounding points of the per-op path (nsr_hashgrid_fwd -> nsr_mlp_vanilla_fwd, nsr_radiance_vanilla_fwd): fp16 operands, fp32
 * accumulation starting from the bias; the density output stays fp32 and sigma = exp(raw0 + density_bias) acts on it; the features
 * enter the colour network rounded to fp16; rgb = sigmoid of the un-rounded fp32 colour output.
 * nsr_bg_field_prepass / _render_fwd: as nsr_nerf_prepass / nsr_nerf_render_fwd; only rows < min(*m_dev or *k_dev, m / k) are read or
 * written.  nsr_bg_field_bwd: as nsr_nerf_field_bwd without row_pos / xyzdir (d_sraw / d_rgb from the unchanged nsr_nerf_ray_bwd);
 * accumulates atomically (caller zeroes) into grad_dmlp [3072], grad_table (table size), grad_dbias [80], grad_cmlp [7168] and
 * grad_cbias [144]; the bias gradients are the column sums of the fp16 pre-activation-gradient tiles, and rows at or past the live count
 * contribute nothing. */
int nsr_bg_field_prepass(const nsr_nerf_t* f, const float* rays, const int32_t* ray_indices, const float* t_starts, const float* t_ends,
                         const void* dmlp_h, const void* table_h, const float* dbias, float* alphas, int64_t m, const int64_t* m_dev,
                         void* stream);
int nsr_bg_field_render_fwd(const nsr_nerf_t* f, const float* rays, const int32_t* ray_indices, const float* t_starts, const float* t_ends,
                            const float* trans, const void* dmlp_h, const void* table_h, const float* dbias, const void* cmlp_h,
                            const float* cbias, void* enc_save_h, float* sigmas, float* rgbs, float* weights, float* acc_rgb, float* opacity,
                            float* depth, int64_t k, const int64_t* k_dev, void* stream);
int nsr_bg_field_bwd(const nsr_nerf_t* f, const float* rays, const int32_t* ray_indices, const float* t_starts, const float* t_ends,
                     const void* enc_save_h, const void* dmlp_h, const float* dbias, const void* cmlp_h, const float* cbias, const float* d_sraw,
                     const float* d_rgb, float* grad_dmlp, float* grad_table, float* grad_dbias, float* grad_cmlp, float* grad_cbias,
                     float loss_scale, const float* amax, int64_t k, const int64_t* k_dev, void* stream);
/* the same backward as TWO launches over the packed inputs (enc_k / d_sraw / d_rgb / xyzdir in packed row order, nsr_pack_kept):
 * (1) network half: recompute + dgrad + wgrad on tensor cores, d(encoding) -> denc_h (f16 [k,32] workspace, still multiplied by the loss
 * scale); (2) table half: a high-occupancy scatter kernel over the same rows -- runs of consecutive samples that share a cell on the
 * coarse levels are summed across the warp before one lane issues the REDs, and x-adjacent corners that are neighbours in memory
 * leave as one 16-byte RED (autograd of tcnn's HashGrid, models/geometry.py:122-130).  Same results as nsr_nerf_field_bwd up to the fp16
 * rounding of d(encoding) and the summation order. */
/* Hopper tensor-core form of the same backward (csrc/nerf_bwd_tc.cu): wgmma.mma_async from shared memory, tile inputs staged by
 * cp.async.bulk (TMA) + mbarrier, warp-specialised GEMM-chain / scatter roles, weight gradients accumulated in shared memory for the
 * whole kernel.  enc_tiles_h = nsr_pack_kept(..., enc_tiled = 1); xyzdir / d_sraw / d_rgb in packed row order; all four
 * buffers readable up to the end of the last 128-row tile.  status (device int, may be NULL): non-zero if a barrier wait timed out. */
int nsr_nerf_field_bwd_tc(const nsr_nerf_t* f, const void* enc_tiles_h, const void* dparams_h, const void* cparams_h, const float* d_sraw,
                          const float* d_rgb, float* grad_dparams, float* grad_cparams, float loss_scale, const float* amax, int64_t k,
                          const int64_t* k_dev, const float* xyzdir, int* status, void* stream);
int nsr_nerf_field_bwd_split(const nsr_nerf_t* f, const void* enc_k_h, const void* dparams_h, const void* cparams_h, const float* d_sraw,
                             const float* d_rgb, float* grad_dparams, float* grad_cparams, float loss_scale, const float* amax, int64_t k,
                             const int64_t* k_dev, const float* xyzdir, void* denc_h, void* stream);
/* The two halves of nsr_nerf_field_bwd_split as separate calls (same arguments; the split form = net followed by scatter with
 * xyz = xyzdir, stride = 6, grad_table = grad_dparams + 3072 = the density network's parameter count, levels [0, 16), ctas_per_sm 0 = 8).
 * denc_h must be 8-byte aligned.  The fused backward scatters level groups in separate launches and zeroes each group's slice of the table
 * right before its launch, so that the slice the REDs hit stays in L2; the data-parallel step also exchanges a finished group beside the
 * next group's scatter.  autograd of tcnn's
 * NetworkWithInputEncoding / Network (models/geometry.py:122-130, models/texture.py:23-30): network half, then the grid backward. */
int nsr_nerf_field_bwd_net(const nsr_nerf_t* f, const void* enc_k_h, const void* dparams_h, const void* cparams_h, const float* d_sraw,
                           const float* d_rgb, float* grad_dparams, float* grad_cparams, float loss_scale, const float* amax, int64_t k,
                           const int64_t* k_dev, const float* xyzdir, void* denc_h, void* stream);
int nsr_nerf_table_scatter(const nsr_grid_t* g, const float* xyz, int32_t stride, const void* denc_h, float loss_scale, const float* amax,
                           float* grad_table, int64_t k, const int64_t* k_dev, int32_t level_begin, int32_t level_end, int32_t ctas_per_sm,
                           void* stream);


/* ---- persistent per-ray kernels (the default fused path) -------------------------------------------------------
 * nsr_nerf_rays_fwd: masks (nsr_march_rays_mask) -> per-ray colour in ONE kernel: a warp owns a ray (atomic ticket queue),
 * walks its samples 32 at a time (gather, density MLP, transmittance scan with the carry in a register, visibility test
 * T >= early_stop_eps, SH4 + colour MLP, weights, per-ray sums) and stops at the first chunk after which T < eps.  Kept
 * samples of ray r land at offsets_m[r] + j, j < kept[r] ("loose" layout).  ticket: device uint32, zero on entry.  Replaces sigma_fn pre-pass + render_visibility
 * + mask compaction + main pass of models/nerf.py:82-109. */
int nsr_nerf_rays_fwd(const nsr_nerf_t* f, const float* rays, const uint32_t* masks, int32_t words, const float* t_min,
                      const int64_t* offsets_m, const int32_t* order, float step, float early_stop_eps, const void* dparams_h,
                      const void* cparams_h,
                      void* enc_save_h, float* sigmas, float* rgbs, float* weights, float* trans, int32_t* kidx, float* acc_rgb,
                      float* opacity, float* depth, int32_t* kept, uint32_t* ticket, int64_t n_rays, const int32_t* counts,
                      const int32_t* bin_counts, int32_t* kept_blocks, void* stream);
/* loose -> packed copy of the kept samples (exact-size ray_indices / t_starts / t_ends / weights of the reference's dict). */
int nsr_pack_kept(const int64_t* offsets_m, const int64_t* offsets_k, const float* t_min, float step, const int32_t* kidx,
                  const float* weights, int32_t* ray_indices_k, float* t_starts_k, float* t_ends_k, float* weights_k /* may be NULL */,
                  int64_t* loose_pos /* packed row -> loose position, may be NULL */,
                  const nsr_nerf_t* f, const float* rays, const void* enc_loose_h /* inputs of the optional outputs below */,
                  void* enc_k_h /* fp16 [K,32] packed copy of the saved encodings, may be NULL */,
                  float* xyzdir_k /* f32 [K,6] unit-cube position + view direction per packed row, may be NULL */,
                  int32_t enc_tiled /* 0: enc_k row-major [K,32]; 1: canonical UMMA tiles of 128 rows (8 KB each; chunk (r, kc) at
                                       ((r/8)*4 + kc)*128 + (r%8)*16 bytes) for nsr_nerf_field_bwd_tc -- enc_k then needs ceil(K/128)*128 rows */,
                  int64_t n_rays, void* stream);
/* nsr_scan_counts(kept) + nsr_pack_kept in one launch: every CTA derives its packed base offset from the kept counts in front of it and
 * writes offsets_k_out [n_rays + 1] for the kernels behind (nsr_nerf_ray_bwd_loose, nsr_nerf_field_bwd's k_dev = offsets_k_out + n_rays). */
int nsr_pack_kept_scan(const int64_t* offsets_m, const int32_t* kept, int64_t* offsets_k_out, const float* t_min, float step,
                       const int32_t* kidx, const float* weights, int32_t* ray_indices_k, float* t_starts_k, float* t_ends_k,
                       float* weights_k, int64_t* loose_pos, const nsr_nerf_t* f, const float* rays, const void* enc_loose_h, void* enc_k_h,
                       float* xyzdir_k, int32_t enc_tiled, int64_t n_rays, const int32_t* kept_blocks, void* stream);
/* (kept_blocks: NULL, or the per-256-ray sums of `kept` that nsr_nerf_rays_fwd accumulated -- the prefix sum then reads <= 32 + 255 values
 * per CTA instead of n_rays.) */
/* compositing backward on the loose layout (same math as nsr_nerf_ray_bwd; t from lattice index + t_min); offsets_k != NULL
 * writes d_sraw / d_rgb in packed row order (row offsets_k[ray] + j) instead of the loose positions. */
int nsr_nerf_ray_bwd_loose(const int64_t* offsets_m, const int32_t* kept, const float* t_min, float step, const int32_t* kidx, const float* trans,
                           const float* weights, const float* sigmas, const float* rgbs, const float* g_rgb, const float* g_opacity,
                           const float* g_depth, const float* g_weights, float* d_sraw, float* d_rgb, float* amax,
                           const int64_t* offsets_k, int64_t n_rays, void* stream);
/* nsr_nerf_rays_bwd: compositing backward + both MLPs + hash scatter in ONE kernel (a warp walks its ray's kept samples 16 at
 * a time from the last chunk to the first carrying the suffix sum).  g_weights is in the loose layout.  amax: device float,
 * zeroed; ticket: device uint32, zeroed; loss_scale <= 0 selects the fp16 dgrad scale on the device from the per-ray
 * gradient bound (t_bound = largest ray parameter, for the depth term). */
int nsr_nerf_rays_bwd(const nsr_nerf_t* f, const float* rays, const float* t_min, const int64_t* offsets_m, const int32_t* kept, float step,
                      const void* enc_save_h, const float* sigmas, const float* rgbs, const float* weights, const float* trans,
                      const int32_t* kidx, const void* dparams_h, const void* cparams_h, const float* g_rgb, const float* g_opacity,
                      const float* g_depth, const float* g_weights, float* grad_dparams, float* grad_cparams, float loss_scale, float* amax,
                      float t_bound, uint32_t* ticket, int64_t n_rays, void* stream);
/* ---- fused NeuS SDF field (VolumeSDF.forward, grad_type 'analytic': models/geometry.py:158-180) -----------------------------
 * points f32 [n,3] world (AABB contraction (x + r) / (2 r)); table fp16 (16 levels, F=2); fp32 VanillaMLP weights of the reference's
 * layout: W1 [64,35] (inputs = [2 x01 - 1 | hash]), b1 [64], W2 [n_out,64], b2 [n_out] (weight-norm already applied), Softplus(beta=100).
 * fwd: sdf [n], grad [n,3] = d sdf / d x_world (analytic), feature [n,n_out] (= the raw network output, sdf in column 0).
 * bwd: upstream g_out [n,n_out], g_sdf [n] (added to column 0) and g_grad [n,3] (each may be NULL) -> grad_table f32 (+=, first AND second order terms, one 8-byte RED per corner),
 * dW1, db1, dW2, db2 (+=).  amax: device float, bound on |g_out|, |g_grad| (fp16 scale of the weight-gradient tiles). */
int nsr_neus_field_fwd(const nsr_grid_t* g, const float* points, const void* table_h, const float* W1, const float* b1, const float* W2,
                       const float* b2, float radius, int32_t n_out, float* sdf, float* grad, float* feature, int64_t n, const int64_t* n_dev,
                       void* stream);
int nsr_neus_field_bwd(const nsr_grid_t* g, const float* points, const void* table_h, const float* W1, const float* b1, const float* W2,
                       const float* b2, float radius, int32_t n_out, const float* g_out, const float* g_sdf, const float* g_grad,
                       const float* amax, float* grad_table, float* dW1, float* db1, float* dW2, float* db2, int64_t n, const int64_t* n_dev,
                       void* stream);
/* The same field under a ProgressiveBandHashGrid level mask: hash levels >= n_active contribute 0 to the features, the analytic normal,
 * every backward term and the table gradient, and are neither gathered nor scattered (their grad_table slices are left untouched, their
 * dW1 columns receive 0).  n_active: device float (clamped to [0, 16], read on the device, so a captured graph follows the schedule).
 * n_active = 16 gives exactly nsr_neus_field_fwd / _bwd. */
int nsr_neus_field_fwd_levels(const nsr_grid_t* g, const float* points, const void* table_h, const float* W1, const float* b1, const float* W2,
                              const float* b2, float radius, int32_t n_out, const float* n_active, float* sdf, float* grad, float* feature, int64_t n,
                              const int64_t* n_dev, void* stream);
int nsr_neus_field_bwd_levels(const nsr_grid_t* g, const float* points, const void* table_h, const float* W1, const float* b1, const float* W2,
                              const float* b2, float radius, int32_t n_out, const float* n_active, const float* g_out, const float* g_sdf,
                              const float* g_grad, const float* amax, float* grad_table, float* dW1, float* db1, float* dW2, float* db2, int64_t n,
                              const int64_t* n_dev, void* stream);
/* ---- fused NeuS SDF field with finite-difference normals + Laplacian (grad_type 'finite_difference': models/geometry.py:181-199) ----
 * Same field and weights as nsr_neus_field_*, evaluated at the centre x_0 = (p + r) / 2r and at the six stencil points
 * (clamp(p +- eps e_a, -r, r) + r) / 2r (true fp32 division); hash levels >= n_active contribute 0 (ProgressiveBandHashGrid mask).
 * fd_state: device float[3] = {eps, fp32(eps^2), n_active} (read on the device, so a captured graph follows the schedule).
 * fwd: sdf [n], feature [n,n_out] at the centre; grad [n,3] = 0.5 (s_a+ - s_a-) / eps and laplace [n] = sum_a (s_a+ + s_a- - 2 sdf) / eps^2.
 *      grad and laplace may both be NULL: centre-only forward.
 * bwd: upstream g_out [n,n_out], g_sdf [n], g_grad [n,3], g_lap [n] (each may be NULL) -> grad_table f32 (+=), dW1, db1, dW2, db2 (+=);
 *      the points get no gradient.  Rows >= *n_dev (when n_dev is non-NULL) are neither read nor written. */
int nsr_neus_field_fd_fwd(const nsr_grid_t* g, const float* points, const void* table_h, const float* W1, const float* b1, const float* W2,
                          const float* b2, float radius, int32_t n_out, const float* fd_state, float* sdf, float* grad, float* feature,
                          float* laplace, int64_t n, const int64_t* n_dev, void* stream);
int nsr_neus_field_fd_bwd(const nsr_grid_t* g, const float* points, const void* table_h, const float* W1, const float* b1, const float* W2,
                          const float* b2, float radius, int32_t n_out, const float* fd_state, const float* g_out, const float* g_sdf,
                          const float* g_grad, const float* g_lap, float* grad_table, float* dW1, float* db1, float* dW2, float* db2, int64_t n,
                          const int64_t* n_dev, void* stream);
/* out[0] = max(|a|, |b|, |c|) over up to three fp32 arrays (NULL / 0 skipped): the bound nsr_neus_field_bwd's amax wants. */
int nsr_absmax3(const float* a, int64_t na, const float* b, int64_t nb, const float* c, int64_t nc, float* out, int64_t rows_cap,
                const int64_t* rows_dev /* non-NULL: arrays are [rows_cap, w] with *rows_dev live rows */, void* stream);

/* sample -> world position / view direction / interval length (models/nerf.py:96-99, models/neus.py:222-225): rays f32 [N,6],
 * positions [K,3] = o + d * (t0 + t1) / 2 (mul then add, no fma), dirs [K,3] and dists [K] = t1 - t0 may be NULL. */
int nsr_sample_points(const float* rays, const int32_t* ray_indices, const float* t_starts, const float* t_ends, float* positions,
                      float* dirs, float* dists, int64_t n, const int64_t* n_dev, void* stream);

/* ---- NeuS shading pieces (models/neus.py:117-139, 225, 237-243) --------------------------------------------------------------
 * (n, n_dev) / (k, k_dev) follow the convention above: non-NULL device count => n is the buffer capacity (CUDA-graph capture).
 * nsr_neus_alpha_fwd: normal = normalize(sdf_grad) and alpha = get_alpha(sdf, normal, dirs, dists) with the cos-anneal ratio;
 * dirs f32 [K,3] per-sample view directions, dists f32 [K] = t_ends - t_starts, inv_s: DEVICE scalar (already clipped to [1e-6, 1e6]);
 * cos_anneal_dev (may be NULL): DEVICE scalar that replaces cos_anneal_ratio, so that a captured graph follows the schedule of
 * models/neus.py:113-115 without re-capture.
 * nsr_neus_alpha_bwd: d_alpha [K], d_normal [K,3] (may be NULL) -> d_sdf [K], d_sdf_grad [K,3], d_inv_s (+=, device scalar). */
int nsr_neus_alpha_fwd(const float* sdf, const float* sdf_grad, const float* dirs, const float* dists, const float* inv_s, float cos_anneal_ratio, const float* cos_anneal_dev, float* alpha, float* normal, int64_t n,
                       const int64_t* n_dev, void* stream);
int nsr_neus_alpha_bwd(const float* sdf, const float* sdf_grad, const float* dirs, const float* dists, const float* inv_s, float cos_anneal_ratio, const float* cos_anneal_dev, const float* d_alpha, const float* d_normal,
                       float* d_sdf, float* d_sdf_grad, float* d_inv_s, int64_t n, const int64_t* n_dev, void* stream);
/* render_weight_from_alpha + accumulate_along_rays x4 (opacity, depth at the sample midpoints, rgb, normal) in one pass per
 * direction.  offsets int64 [n_rays+1]; comp_normal is the un-normalised weighted sum.  Backward: any of the g_* may be NULL. */
int nsr_neus_composite_fwd(const float* alphas, const float* rgbs, const float* normals, const float* t_starts, const float* t_ends,
                           const int64_t* offsets, float* weights, float* trans, float* opacity, float* depth, float* comp_rgb,
                           float* comp_normal, int64_t n_rays, void* stream);
int nsr_neus_composite_bwd(const float* alphas, const float* rgbs, const float* normals, const float* t_starts, const float* t_ends,
                           const float* weights, const float* trans, const int64_t* offsets, const float* g_weights,
                           const float* g_opacity, const float* g_depth, const float* g_rgb, const float* g_normal, float* d_alphas,
                           float* d_rgbs, float* d_normals, int64_t n_rays, void* stream);
/* VolumeRadiance (see nsr_radiance_t): feat f32 [n,n_feat], dirs f32 [n,3] (unit view directions, per sample), extra f32 [n,n_extra] (or NULL), params fp16 [7168] in tcnn order,
 * rgb f32 [n,3].  Backward: d_rgb [n,3] -> d_feat, d_extra (either may be NULL), grad_params f32 [7168] (+=);
 * loss_scale <= 0: choose the fp16 dgrad scale from *amax (device float: max |d_rgb|). */
int nsr_radiance_fwd(const nsr_radiance_t* p, const float* feat, const float* dirs, const float* extra,
                     const void* params_h, float* rgb, int64_t n, const int64_t* n_dev, void* stream);
int nsr_radiance_bwd(const nsr_radiance_t* p, const float* feat, const float* dirs, const float* extra,
                     const void* params_h, const float* d_rgb, float loss_scale, const float* amax, float* d_feat, float* d_extra,
                     float* grad_params, int64_t n, const int64_t* n_dev, void* stream);
/* The same module when its network is the reference's VanillaMLP (models/network_utils.py:95-139; configs/neus-dtu.yaml:58-70
 * texture, :93-105 texture_bg: ReLU, 64 neurons, two hidden layers, biases, fp32 output, computed under autocast(False)):
 * n_feat + 16 + n_extra <= 32 (narrower inputs are zero padded), weights_h fp16 [7168] = W1 [64,32] (columns beyond the input
 * width zero) | W2 [64,64] | W3 [16,64] (rows 3.. zero), bias f32 [144] = b1 | b2 | b3 (padded to 16); fp16 tensor-core operands,
 * fp32 accumulation starting from the bias, fp32 output (act_mode 0 none, 1/2 sigmoid).  Backward adds grad_weights f32 [7168] (+=)
 * and grad_bias f32 [144] (+=). */
int nsr_radiance_vanilla_fwd(const nsr_radiance_t* p, const float* feat, const float* dirs, const float* extra, const void* weights_h,
                             const float* bias, float* rgb, int64_t n, const int64_t* n_dev, void* stream);
int nsr_radiance_vanilla_bwd(const nsr_radiance_t* p, const float* feat, const float* dirs, const float* extra, const void* weights_h,
                             const float* bias, const float* d_rgb, float loss_scale, const float* amax, float* d_feat, float* d_extra,
                             float* grad_weights, float* grad_bias, int64_t n, const int64_t* n_dev, void* stream);

/* ---- training-batch front end (SURVEY 8f-3; preprocess_data of systems/nerf.py:33-91 / systems/neus.py:34-96 + models/ray_utils.py:23-43)
 * ray r comes from image index[r], pixel (x[r], y[r]) (index == NULL: image fixed_index, pixel (r % W, r / W): a whole image in
 * row-major order).  directions f32 [H,W,3] (dirs_per_image 0) or [n_images,H,W,3] (1); c2w f32 [n_images, c2w_rows (3|4), 4];
 * rays f32 [n,6] = c2w[:,3] | normalize(sum_j directions_j * c2w[i][j]) (F.normalize, eps 1e-12).  Optional (NULL = skip):
 * rgb f32 [n,3] = images[index,y,x,:3] (images f32 [n_images,H,W,channels]), fg f32 [n] = masks[index,y,x] (masks f32
 * [n_images,H,W]); apply_mask: rgb = rgb * fg + bg * (1 - fg), bg f32 [3].  Out-of-range indices are clamped. */
int nsr_gather_rays(const float* directions, int32_t dirs_per_image, const float* c2w, int32_t c2w_rows, const float* images,
                    int32_t channels, const float* masks, const int64_t* index, const int64_t* x, const int64_t* y, int32_t fixed_index,
                    const float* bg, int32_t apply_mask, int32_t H, int32_t W, int32_t n_images, float* rays, float* rgb, float* fg,
                    int64_t n, void* stream);

/* ---- isosurface extraction (SURVEY 8f-4; models/geometry.py:32-112: MarchingCubeHelper + isosurface_; replaces the host copy of the
 * level grid and the single-core PyMCubes call).  field f32 [nx,ny,nz] (z fastest = torch.meshgrid(indexing='ij').reshape(-1));
 * INSIDE <=> value > iso, value = negate ? -field : field (the reference hands -level to mcubes: geometry.py:62).
 *   nsr_mc_count: block_offsets int32 [2 * B], B = ceil(nx*ny*nz / 256): on return the exclusive prefix sums of the per-block vertex
 *                 counts ([0,B)) and triangle counts ([B,2B)); totals int64 [2] (device) = (V, F).  The caller reads totals (one host
 *                 sync), allocates verts f32 [V,3] and faces int64 [F,3], then
 *   nsr_mc_emit:  vid_map int32 [nx*ny*nz] workspace; verts = (index coordinate / (n-1)) * (hi - lo) + lo per axis (lo, hi: HOST
 *                 float[3], the box the grid spans); vertices in (grid point, axis) order, triangles in (cell, case-table) order,
 *                 wound so that their normals point to the outside (smaller values).  Deterministic, no atomics.
 * The case table (csrc/mc_table.inc) is generated by mc_table.py with one fixed rule for ambiguous faces => no holes. */
int nsr_mc_count(const float* field, int32_t nx, int32_t ny, int32_t nz, float iso, int32_t negate, int32_t* block_offsets, int64_t* totals,
                 void* stream);
int nsr_mc_emit(const float* field, int32_t nx, int32_t ny, int32_t nz, float iso, int32_t negate, const int32_t* block_offsets,
                const float* lo, const float* hi, int32_t* vid_map, float* verts, int64_t n_verts, int64_t* faces, int64_t n_faces,
                void* stream);

/* ---- gradient exchange over NVLink peer memory (SURVEY 8e; replaces the NCCL all-reduce of Lightning DDP, launch.py:98) ---------
 * Every rank holds its flat fp32 gradient vector in a peer-mapped (symmetric) buffer of n floats (n % 4 == 0).
 * nsr_p2p_barrier: all-ranks barrier on the stream: flags = one peer-mapped int32[>= world] array per rank (zeroed once),
 *   flag_ptrs_host[q] = address of rank q's array in THIS process; epoch_dev / err_dev: local device int32 (zeroed once;
 *   *err_dev becomes 1 if a peer never arrived within the spin bound).
 * nsr_p2p_allreduce_mean: in-place mean over the ranks; rank r reduces chunk r (P2P loads from peer_ptrs_host[q], or one
 *   multimem.ld_reduce on multicast_ptr when the buffer has an NVSwitch multicast mapping) and writes it into every replica.
 *   Must be bracketed by barriers: barrier, allreduce, barrier. */
int nsr_p2p_barrier(const uint64_t* flag_ptrs_host, int32_t* epoch_dev, int32_t* err_dev, int32_t rank, int32_t world, void* stream);
int nsr_p2p_allreduce_mean(const uint64_t* peer_ptrs_host, void* multicast_ptr, int32_t rank, int32_t world, int64_t n, void* stream);
/* nsr_p2p_exchange_mean (reference: the gradient all-reduce Lightning DDP inserts, launch.py:98 `strategy='ddp'`): the same exchange as ONE launch -- entry barrier, reduce-scatter + all-gather, exit barrier inside the kernel
 *   (what one bucket of DDP's all-reduce is, launch.py:98).  flag arrays need 64 int32 per rank (entry epochs in [32,48), exit epochs in
 *   [48,64); [0,16) stays nsr_p2p_barrier's); epoch_counter_dev: local int32[2] {last completed epoch, CTA counter}, zeroed once.  No surrounding barriers needed;
 *   graph-replay safe (the epoch is device state).  When it returns on the stream, every replica holds the mean and no peer reads
 *   this rank's buffer any more. */
int nsr_p2p_exchange_mean(const uint64_t* peer_ptrs_host, const uint64_t* flag_ptrs_host, void* multicast_ptr, int32_t* epoch_counter_dev,
                          int32_t* err_dev, int32_t rank, int32_t world, int64_t n, void* stream);
/* the same over floats [begin, begin + count) of the buffer (both multiples of 4 * world), on `channel` (0..3: own flag slots
 * [32 + 32 channel, 64 + 32 channel) of a 256-int32 flag array and own epoch_counter_dev pair) so that exchanges of different ranges may be
 * in flight at the same time on different streams; ctas_per_sm: 0 = default. */
int nsr_p2p_exchange_mean_range(const uint64_t* peer_ptrs_host, const uint64_t* flag_ptrs_host, void* multicast_ptr, int32_t* epoch_counter_dev,
                                int32_t* err_dev, int32_t rank, int32_t world, int64_t begin, int64_t count, int32_t channel, int32_t ctas_per_sm,
                                void* stream);

/* ---- occupancy-grid refresh (SURVEY 8f-1; nerfacc OccupancyGrid._update behind every_n_step: models/nerf.py:45-55,
 * models/neus.py:79-111).  The caller draws the cells (int64 flat indices ix*R*R + iy*R + iz; NULL = every cell once) and the
 * in-cell jitter U[0,1)^3, evaluates its occ function on the returned world points, then:
 *   update:   occs[cell] = max(occs[cell] * ema_decay, occ)   (duplicates: max of their values), partial = per-block sums of occs
 *             scratch: f32 [n_cells] work grid (sparse updates only); partial: f64 [1024]
 *   binarize: binary (u8 [n_cells], may be NULL) = occs > min(mean(occs), occ_thre); bits = packed bitfield (bit idx&31 of word
 *             idx>>5), coarse_bits (may be NULL; res % 4 == 0) = "any bit in the 4^3 block" over (res/4)^3 cells.
 * p: only roi, res and contraction (0 AABB, 2 UN_BOUNDED_SPHERE: valid[i] = 0 outside the unit ball) are read. */
int nsr_occgrid_points(const nsr_march_t* p, const int64_t* cells, const float* jitter, float* x_world, uint8_t* valid, int64_t n,
                       void* stream);
int nsr_occgrid_update(float* occs, const int64_t* cells, const float* occ, float* scratch, float ema_decay, double* partial, int64_t n,
                       int64_t n_cells, void* stream);
int nsr_occgrid_binarize(const float* occs, const double* partial, float occ_thre, uint8_t* binary, uint32_t* bits, uint32_t* coarse_bits,
                         int32_t res, int64_t n_cells, void* stream);

/* ---- optimizer (SURVEY 8f-2; systems/utils.py:314-325) ------------------------------------------------------------------------
 * One fused pass of torch.optim.AdamW over a flat fp32 vector: un-scale, skip on *found_inf != 0, decoupled weight decay, moments,
 * update, and (params_half != NULL) the fp16 copy the kernels read.  dev_lr_step (device float[2] = {lr, step}, or NULL)
 * overrides h->lr / h->step for CUDA-graph capture.  All buffers 16-byte aligned. */
int nsr_adamw_step(const nsr_adamw_t* h, float* params, const float* grads, float* exp_avg, float* exp_avg_sq, void* params_half,
                   const float* dev_lr_step, const float* found_inf, int64_t n, void* stream);
/* found_inf[0] = 1 if any entry of grads is inf / nan (left untouched otherwise). */
int nsr_grad_nonfinite(const float* grads, float* found_inf, int64_t n, void* stream);

/* ---- training-step back end (SURVEY 8f-3; systems/nerf.py:68-97) ---------------------------------------------------
 * background blend + masked smooth-L1 over the valid rays: comp = acc_rgb + bg (1 - opacity), valid = opacity > 0,
 * loss = sum smooth_l1(comp - target) / max(3 n_valid, 1).  accum: device float[4], zeroed by the entry point:
 * [0] loss sum, [1] n_valid, [2] the loss (written by a one-thread epilogue); comp_rgb [n,3] optional output.
 * The backward writes dL/d acc_rgb and dL/d opacity. */
int nsr_nerf_loss_fwd(const float* acc_rgb, const float* opacity, const float* bg3, const float* target, float* comp_rgb, float* accum2,
                      int64_t n_rays, void* stream);
int nsr_nerf_loss_bwd(const float* acc_rgb, const float* opacity, const float* bg3, const float* target, const float* accum2,
                      const float* g_loss, float* g_acc_rgb, float* g_opacity, int64_t n_rays, void* stream);
/* NeuS losses (systems/neus.py:98-121): comp_rgb [N,3] (= comp_rgb_full), valid u8 [N] (= rays_valid_full), target [N,3],
 * opacity [N], fg_mask f32 [N] (NULL: no mask loss), sdf_grad [K,3] (eikonal; NULL skips), sdf [K] (sparsity; NULL skips).
 * fwd: accum8 = device float[8] work (zeroed here), losses7 = {rgb_mse, rgb_l1, eikonal, mask, opaque, sparsity, weighted total};
 * the rgb means run over the valid rays (denominator clamped to >= 1).  bwd: d total / d inputs times *g_loss (NULL = 1);
 * g_sdf_grad / g_sdf may be NULL. */
int nsr_neus_loss_fwd(const nsr_neus_loss_t* p, const float* comp_rgb, const uint8_t* valid, const float* target, const float* opacity,
                      const float* fg_mask, const float* sdf_grad, const float* sdf, float* accum8, float* losses7, int64_t n_rays,
                      int64_t k, const int64_t* k_dev, void* stream);
int nsr_neus_loss_bwd(const nsr_neus_loss_t* p, const float* comp_rgb, const uint8_t* valid, const float* target, const float* opacity,
                      const float* fg_mask, const float* sdf_grad, const float* sdf, const float* accum8, const float* g_loss,
                      float* g_comp_rgb, float* g_opacity, float* g_sdf_grad, float* g_sdf, int64_t n_rays, int64_t k, const int64_t* k_dev,
                      void* stream);
/* Distortion loss of mip-NeRF 360 (torch_efficient_distloss.flatten_eff_distloss; systems/nerf.py:103-106, systems/neus.py:131-139) over
 * n packed samples sorted by ray: loss = sum_rays [sum_ij w_i w_j |m_i - m_j| + 1/3 sum_i w_i^2 d_i] / (ray_ids[last live row] + 1).
 * w_pos (int64 [n], may be NULL): the weight of row i is w[w_pos[i]] and its gradient goes to g_w[w_pos[i]].  t_mode 0: a = midpoints,
 * b = intervals; t_mode 1: a = t_starts, b = t_ends.  n_dev (device int64, may be NULL): live row count; rows at or past it are never
 * read or written.  fwd: accum2 = device float[2], zeroed here; [1] = the loss (0 for no live rows).  bwd: g_w at every live row =
 * *g_loss (NULL = 1) * dloss/dw, plain stores (no other entry of g_w is written).  Neither synchronises with the host. */
int nsr_distortion_fwd(const float* w, const int64_t* w_pos, const float* a, const float* b, int32_t t_mode, const int32_t* ray_ids,
                       float* accum2, int64_t n, const int64_t* n_dev, void* stream);
int nsr_distortion_bwd(const float* w, const int64_t* w_pos, const float* a, const float* b, int32_t t_mode, const int32_t* ray_ids,
                       const float* g_loss, float* g_w, int64_t n, const int64_t* n_dev, void* stream);

#ifdef __cplusplus
}
#endif
#endif
