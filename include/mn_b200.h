/*
 * mn_b200.h — C ABI of the Mega-NeRF rendering hot path for H100 (sm_90a; libmn_b200.so).
 *
 * The reference (cmusatyalab/mega-nerf @76d8d76b) is pure Python/PyTorch and has NO FFI / plugin
 * boundary of its own (SURVEY.md §8b); this header defines the boundary underneath the Python call
 * surface it does have.  Each entry point cites the reference code it replaces (file:line, relative
 * to the reference repository root).  The Python host mirror lives in mega_nerf_b200/*.py and binds
 * these symbols with ctypes (see INTEGRATION.md).
 *
 * Conventions
 *  - every pointer named *_d is a DEVICE pointer to fp32 (or int32 where stated), row-major, borrowed
 *    for the duration of the call; nothing is retained except by mn_model_set_weights (see there);
 *  - `stream` is a cudaStream_t passed as void* (torch.cuda.current_stream().cuda_stream); all work is
 *    enqueued on it, no entry point synchronises the host unless stated;
 *  - every function returns MN_OK or an MN_ERR_* code; mn_last_error(ctx) gives the message.  Error
 *    texts for the two reference exceptions are the reference's own (nerf.py:121-123,
 *    rendering.py:412-414) so the Python shim can re-raise `Exception(msg)` verbatim;
 *  - entry points are thread-safe per context, keep no hidden global state and spawn no threads.
 */
#ifndef MN_B200_H
#define MN_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MN_ABI_VERSION 1

enum {
    MN_OK = 0,
    MN_ERR_INVALID = 1,    /* bad argument */
    MN_ERR_CUDA = 2,       /* a CUDA runtime call or launch failed */
    MN_ERR_SHAPE = 3,      /* "Unexpected input shape: ..."                (models/nerf.py:121-123) */
    MN_ERR_SPHERE = 4,     /* "Not all your cameras are bounded by ..."    (rendering.py:412-414)  */
    MN_ERR_WORKSPACE = 5,  /* workspace too small */
    MN_ERR_UNSUPPORTED = 6 /* configuration outside what the kernels cover */
};

/* Arithmetic of the MLP stage. */
enum {
    MN_PREC_FP32 = 0,      /* CUDA-core fp32 FMA, parity mode (<= 1e-5 of the fp32 oracle)              */
    MN_PREC_TC_F16 = 1,    /* wgmma, fp16 operands, fp32 register accumulate, 1 MMA pass                */
    MN_PREC_TC_F16X3 = 2   /* wgmma, hi/lo fp16 split of both operands, 3 MMA passes per algorithmic    */
};

typedef struct mn_ctx mn_ctx;
typedef struct mn_model mn_model;

/* ---- context --------------------------------------------------------------------------------- */
int mn_abi_version(void);
int mn_create(mn_ctx** out, int device);
void mn_destroy(mn_ctx* ctx);
const char* mn_last_error(const mn_ctx* ctx);
/* Device-side status word written by kernels that detect reference exceptions (sphere check) or
 * capacity overflow; mn_check_status copies it back (this one DOES synchronise `stream`) and maps it
 * to MN_ERR_SPHERE / MN_ERR_WORKSPACE.  Call it where the reference has its own host sync
 * (rendering.py:412 `.any()`).  */
int mn_check_status(mn_ctx* ctx, void* stream);

/* Measurement hooks used by bench.py: number of kernels launched through this context so far, and
 * CUDA-event timing (on the launching stream) of the MLP-stage kernel launches. */
long long mn_launch_count(const mn_ctx* ctx);
int mn_profile_enable(mn_ctx* ctx, int on);
int mn_profile_read(mn_ctx* ctx, double* total_ms, long long* n_launches);

/* ---- ray generation --------------------------------------------------- mega_nerf/ray_utils.py */
/* get_ray_directions (ray_utils.py:6-18): out_d [H*W*3]. */
int mn_ray_directions(mn_ctx* ctx, int W, int H, float fx, float fy, float cx, float cy, int center_pixels,
                      float* out_d, void* stream);
/* get_rays / get_rays_batch / _get_rays_inner / _truncate_with_plane_intersection
 * (ray_utils.py:21-84).  dirs_d [n_dirs_sets? P*3] with dirs_batched!=0 meaning [n,P,3];
 * c2w_d [n,3,4]; out_d [n,P,8] = (o3,d3,near,far). */
int mn_rays(mn_ctx* ctx, const float* dirs_d, int dirs_batched, const float* c2w_d, int n_poses, int64_t P,
            float near, float far, int has_altitude, float alt_max, float alt_min, float* out_d, void* stream);

/* The loader's use of get_rays_batch (mega_nerf/datasets/filesystem_dataset.py:109-124; SURVEY.md §8f-6): one ray per
 * (image, pixel) pair of a training chunk.  The reference computes the full [#unique images, #unique pixels, 8] product on
 * the device, copies it to the host (`.cpu()`, :121) and gathers the pairs there (:125); this entry computes the M pairs only.
 *   dirs_d [P,3] (the shared direction table, :40-47); c2w_d [n_poses,3,4]; img_idx_d / pix_idx_d int32 [M] (row of c2w_d /
 *   row of dirs_d); out_d [M,8].  An index outside its table raises MN_ERR_INVALID at the next mn_check_status (the
 *   reference's fancy indexing raises IndexError) and the ray is NaN. */
int mn_rays_pairs(mn_ctx* ctx, const float* dirs_d, int64_t P, const float* c2w_d, int n_poses, const int32_t* img_idx_d,
                  const int32_t* pix_idx_d, int64_t M, float near, float far, int has_altitude, float alt_max, float alt_min,
                  float* out_d, void* stream);

/* ---- training batches -------------------- DataLoader(FilesystemDataset / MemoryDataset), runner.py:228-238 */
/* One training batch from a device-resident chunk (mega_nerf_b200/batches.py): dst_k[b] = src_k[idx_d[b]] for up to three
 * row-major columns of 4-byte elements (rgbs [n,3] fp32, rays [n,8] fp32, img_indices [n] int32), what the reference's
 * DataLoader assembles row by row with `__getitem__` + `default_collate`.
 *   idx_d int64 [B] (a slice of the permutation, already on the device); n_rows = rows of the chunk; src_k_d [n_rows, w_k],
 *   dst_k_d [B, w_k]; a column with src_k_d == NULL is skipped.  Rows move in 16-byte units where w_k % 4 == 0 and both
 *   pointers are 16-byte aligned.  One launch on `stream`, no host sync.  An index outside [0, n_rows) is never read: its
 *   output row is all one bits and MN_ERR_INVALID is raised at the next mn_check_status. */
int mn_gather_batch(mn_ctx* ctx, const int64_t* idx_d, int64_t B, int64_t n_rows, const void* src0_d, int w0, void* dst0_d,
                    const void* src1_d, int w1, void* dst1_d, const void* src2_d, int w2, void* dst2_d, void* stream);

/* ---- sampling --------------------------------------------------------- mega_nerf/rendering.py */
/* Coarse depths + optional stratified jitter + points (rendering.py:82-87, 472-483).
 *   rays_d [N,8]; z_steps_d [S] (torch.linspace(0,1,S) — passed in, never restated, SURVEY §8c);
 *   far_d optional [N] override of rays[:,7] (fg_far clamp, rendering.py:45);
 *   rand_d optional [N,S] U[0,1) draws, used iff perturb>0;  z_out_d [N,S]; xyz_out_d [N,S,3]. */
int mn_sample_coarse(mn_ctx* ctx, const float* rays_d, const float* far_d, const float* z_steps_d,
                     const float* rand_d, float perturb, int64_t N, int S, float* z_out_d, float* xyz_out_d,
                     void* stream);
/* Stratified expansion of a shared 1-D depth vector (background path, rendering.py:47-50). */
int mn_stratify(mn_ctx* ctx, const float* z_d, int64_t z_row_stride, const float* rand_d, float perturb, int64_t N,
                int S, float* z_out_d, void* stream);
/* xyz = o + d*z, separately rounded mul and add (rendering.py:100 lambda, :223). */
int mn_points_from_z(mn_ctx* ctx, const float* rays_d, const float* z_d, int64_t N, int S, float* xyz_out_d,
                     void* stream);
/* _sample_pdf / _sample_cdf (rendering.py:486-536).  Exactly one of weights_d / cdf_d is given:
 *   weights_d [N, w_stride] is the FULL coarse weight row; columns 1..S-2 are used (rendering.py:215);
 *   cdf_d [N,S-2] is an externally supplied cdf (stage test: indices are bit-exact given cdf and u);
 *   z_coarse_d [N,S] (bins are its midpoints, rendering.py:213);  u_d [F] (u_row_stride=0) or [N,F];
 *   z_out_d [N,F]; inds_out_d optional int64 [N,F]; cdf_out_d optional [N,S-2]. */
int mn_sample_pdf(mn_ctx* ctx, const float* z_coarse_d, const float* weights_d, int64_t w_stride,
                  const float* cdf_d, const float* u_d, int64_t u_row_stride, int64_t N, int S, int F,
                  float* z_out_d, int64_t* inds_out_d, float* cdf_out_d, void* stream);
/* Per-ray sort of cat[a, b] (ascending, or descending) — cascade resample merge (rendering.py:219). */
int mn_sort_cat(mn_ctx* ctx, const float* a_d, int na, const float* b_d, int nb, int64_t N, int descending,
                float* out_d, void* stream);

/* Volume rendering (rendering.py:336-393).  One warp per ray.
 *   own samples: raw_d [N,S,4] = (r,g,b,sigma) and z_d [N,S] of THIS pass (already flipped if flip);
 *   optional stored coarse samples to merge with (non-cascade fine pass, rendering.py:336-350):
 *     raw2_d [N,S2,4], z2_d [N,S2] (and depth_real2_d) — sorted together by z, descending iff flip;
 *   last_delta_d [N]: 1e10, or the sphere-exit depth for rays that continue into the background; when
 *     < 1e10 the max of the pass's OWN z is subtracted first (rendering.py:191-193,224-225; quirk Q5);
 *   depth_real_d optional [N,S]: background real depths used for the depth outputs.
 *   outputs (any may be NULL): weights [N,S+S2] (merged order), rgb [N,3], depth [N], depth_var [N],
 *   bg_lambda [N]. */
int mn_composite(mn_ctx* ctx, const float* raw_d, const float* z_d, const float* depth_real_d, int S,
                 const float* raw2_d, const float* z2_d, const float* depth_real2_d, int S2,
                 const float* last_delta_d, int64_t N, int flip,
                 float* weights_out_d, float* rgb_out_d, float* depth_out_d, float* depth_var_out_d,
                 float* bg_lambda_out_d, void* stream);

/* Background geometry (rendering.py:396-469).
 * mn_intersect_sphere: fg_far [N]; raises the device status MN_ERR_SPHERE when a camera lies outside. */
int mn_intersect_sphere(mn_ctx* ctx, const float* rays_d, const float* center3_d, const float* radius3_d, int64_t N,
                        float* fg_far_out_d, void* stream);
/* mn_points_outside: for rays selected by ray_ids_d (int64 [n], or NULL = all), inverse depths
 * depth_d [n,S] -> pts [n,S,4] (or [n,S,7] with the real-xyz routing prefix) and depth_real [n,S]. */
int mn_points_outside(mn_ctx* ctx, const float* rays_d, const int64_t* ray_ids_d, const float* depth_d,
                      const float* center3_d, const float* radius3_d, int64_t n, int S, int include_xyz_real,
                      int cluster_2d, float* pts_out_d, float* depth_real_out_d, void* stream);

/* eval_sh + sigmoid (spherical_harmonics.py:55-106, rendering.py:301-306).
 *   coef_d [B, coef_stride]: first 3*(deg+1)^2 columns are channel-major SH coefficients, column
 *   3*(deg+1)^2 is sigma (copied through);  dirs_d [B/dir_div, 3];  out_d [B,4]. */
int mn_sh_to_rgb(mn_ctx* ctx, int deg, const float* coef_d, int64_t coef_stride, const float* dirs_d,
                 int64_t dir_stride, int dir_div, int64_t B, int apply_sigmoid, float* out_d, void* stream);
/* Embedding.forward (models/nerf.py:8-25): x [B,dim] -> [B, dim*(1+2*n_freqs)]. */
int mn_embed(mn_ctx* ctx, const float* x_d, int64_t B, int dim, int n_freqs, float* out_d, void* stream);

/* ---- networks --------------------------------------------------------- mega_nerf/models/*.py */
typedef struct {
    int kind;              /* 0 = NeRF (nerf.py:45), 1 = Cascade (cascade.py:7; sub 0 coarse, 1 fine),
                              2 = MegaNeRF (mega_nerf.py:7; n_sub sub-modules)                        */
    int n_sub;
    int pos_xyz_dim, pos_dir_dim, layers, layer_dim, appearance_dim, affine_appearance, appearance_count,
        rgb_dim, xyz_dim, shifted_softplus;
    int n_skip;
    int skip_layers[8];
    float boundary_margin; /* MegaNeRF only */
    int xyz_real;          /* MegaNeRF only: first 3 input columns are routing-only (mega_nerf.py:36) */
    int cluster_dim_start; /* MegaNeRF only: 1 if cluster_2d */
} mn_model_desc;

/* fp32 device tensors of one NeRF sub-module, in the reference state-dict layout ([out,in] row-major). */
typedef struct {
    const float* xyz_w[16];
    const float* xyz_b[16];
    const float *sigma_w, *sigma_b, *final_w, *final_b, *dir_a_w, *dir_a_b, *rgb_w, *rgb_b, *embedding_a,
        *affine_w, *affine_b;
} mn_nerf_weights;

int mn_model_create(mn_ctx* ctx, const mn_model_desc* desc, mn_model** out);
void mn_model_destroy(mn_model* m);
/* centroids [n_sub,3] device fp32; copied. */
int mn_model_set_centroids(mn_model* m, const float* centroids_d, void* stream);
/* (Re)pack one sub-module: transposes / pads / splits the weights into model-owned device buffers
 * (the only persistent allocation the library makes).  Call again whenever the parameters change. */
int mn_model_set_weights(mn_model* m, int sub, const mn_nerf_weights* w, void* stream);

/* Where the per-row model inputs come from.  Mirrors the two ways the reference builds rows:
 *   mode 0 — an explicit row matrix x [B, cols] as handed to nn.Module.__call__ (nerf.py:115);
 *   mode 1 — ray-structured: xyz [B, xyz_cols] plus per-ray directions / image indices that the
 *            reference would broadcast with repeat+cat (rendering.py:275-292,311-319): row b belongs
 *            to ray b / samples_per_ray. */
typedef struct {
    int mode;
    const float* x_d;       /* mode 0: [B, cols]; mode 1: xyz [B, xyz_cols]                          */
    int cols;               /* mode 0: cols; mode 1: xyz_cols (3, 4, or 7 with the real-xyz prefix)  */
    const float* dirs_d;    /* mode 1: [n_rays, dir_stride], NULL if the model takes no dirs          */
    int64_t dir_stride;
    const float* idx_d;     /* mode 1: [n_rays] image indices as fp32, NULL if no appearance          */
    int samples_per_ray;    /* mode 1 */
} mn_rows;

/* Slot capacity per row reserved for blended routing (boundary_margin > 1): a row within the margin
 * of more sub-modules than this raises MN_ERR_WORKSPACE at the next mn_check_status.  Default
 * min(n_sub, 4); hard routing always uses 1. */
int mn_model_set_max_multiplicity(mn_model* m, int max_multiplicity);

size_t mn_model_workspace_bytes(const mn_model* m, int64_t B, int precision);
/* nn.Module.__call__(x, sigma_only, sigma_noise) for NeRF / Cascade(use_coarse) / MegaNeRF
 * (nerf.py:115-160, cascade.py:13-18, mega_nerf.py:19-61).  out_d [B, out_cols] with
 * out_cols = 1 if sigma_only else rgb_dim+1.  sigma_noise_d optional [B].  Returns MN_ERR_SHAPE with
 * the reference's message on a bad column count. */
int mn_model_forward(mn_ctx* ctx, mn_model* m, const mn_rows* rows, int64_t B, int use_coarse, int sigma_only,
                     const float* sigma_noise_d, int precision, float* out_d, void* workspace_d,
                     size_t workspace_bytes, void* stream);
/* Routing only (mega_nerf.py:21-30), for the stage tests: assign_out_d int32 [B] (margin==1) or
 * weights_out_d [B,n_sub] (margin>1). */
int mn_model_route(mn_ctx* ctx, mn_model* m, const mn_rows* rows, int64_t B, int32_t* assign_out_d,
                   float* weights_out_d, void* stream);
/* Density grid of octree extraction (scripts/create_octree.py:61-105 _auto_scale, :139-162 _step1): sigma_out_d[r - row0] is
 * nerf(x_r, sigma_only=True) (Cascade: nerf(use_coarse, x_r, ...)) for every lattice row r in [row0, row0 + n_rows) of the
 * reso^3 lattice torch.stack(torch.meshgrid(xx, yy, zz)).reshape(3, -1).T, i.e. r = (i * reso + j) * reso + k (x slowest) and
 * x_r = (((i, j, k) + 0.5) / reso - offset) / scale per axis in fp32, bit-identical to torch's CPU lattice.  The range runs
 * through slabs of a fixed row count - lattice points into the workspace, then the mn_model_forward kernels (sigma_only,
 * `precision`) - on `stream`, with no allocation and no host sync; the workspace size does not depend on reso or n_rows.
 * Routing slots are sized for every sub-module per row (a dense box reaches past the centroid hull), for this call only.
 * As with any model call, a tail slab of <= 25 rows routes through cdist's direct path (mn_model_route).
 *   reso 1 .. 2097151; scale > 0 on every axis; the range inside reso^3 (else MN_ERR_INVALID); models whose rows are not plain
 *   xyz (xyz_dim != 3, or a real-xyz routing prefix) return MN_ERR_UNSUPPORTED. */
size_t mn_model_density_grid_workspace_bytes(const mn_model* m, int precision);
int mn_model_density_grid(mn_ctx* ctx, mn_model* m, int use_coarse, const float offset[3], const float scale[3], int reso,
                          int64_t row0, int64_t n_rows, int precision, float* sigma_out_d, void* workspace_d,
                          size_t workspace_bytes, void* stream);
/* Counters of the last mn_model_forward on this model, read back lazily (synchronises `stream`):
 * slots = routed (row, sub-module) pairs, tiles = 128-row MLP tiles. */
int mn_model_last_stats(mn_ctx* ctx, mn_model* m, int64_t* slots, int64_t* tiles, void* stream);

/* ---- the whole foreground path in one call ------------------------------ mega_nerf/rendering.py:15-248 ----
 * render_rays(nerf, bg_nerf=None, ...) in eval mode (no jitter, no density noise): coarse depths -> query -> weights ->
 * inverse-CDF resampling -> fine query -> merge + volume rendering, sequenced on `stream` from the caller's workspace
 * (mn_render_rays_workspace_bytes) with no allocation and no host sync.  Same results as the stage entry points called
 * one by one (that is what it does).
 *   rays_d [N,8]; image_indices_d [N] fp32 (required iff the model has an appearance embedding);
 *   z_steps_d [coarse_samples] and u_fine_d [fine_samples] = torch.linspace(0,1,.) passed in (SURVEY §8c);
 *   use_cascade must match the model kind (Cascade <-> 1); sh_deg = -1 for a plain rgb head;
 *   outputs: rgb_out_d [N,3] = rgb_fine (rgb_coarse when fine_samples == 0); depth_out_d / depth_var_out_d optional [N];
 *   rgb_coarse_out_d optional [N,3], written under use_cascade with fine_samples > 0 (rendering.py:199). */
size_t mn_render_rays_workspace_bytes(const mn_model* m, int64_t N, int coarse_samples, int fine_samples, int use_cascade,
                                      int sh_deg, int precision);
int mn_render_rays(mn_ctx* ctx, mn_model* m, const float* rays_d, const float* image_indices_d, int64_t N,
                   const float* z_steps_d, int coarse_samples, const float* u_fine_d, int fine_samples, int use_cascade,
                   int sh_deg, int precision, float* rgb_out_d, float* depth_out_d, float* depth_var_out_d,
                   float* rgb_coarse_out_d, void* workspace_d, size_t workspace_bytes, void* stream);

/* ---- the same with a background (NeRF++) network ------------------------ mega_nerf/rendering.py:15-173 ----
 * render_rays(nerf, bg_nerf, ...) in eval mode: the sphere split of every ray (fg_far = max(exit of the ellipsoid
 * sphere_center3 / sphere_radius3, near); a ray reaches the background iff far > fg_far), the background pass over those rays
 * (compacted on the device in ascending ray order; half the coarse samples, fine_samples / 2 draws, points inside the
 * inverted sphere, flipped two-pass render), the foreground pass (far clipped to fg_far, last delta fg_far) and the blend
 * val + bg_val * bg_lambda.  No host sync: the background ray count stays on the device, every background kernel skips the
 * rays past it, so the launch sequence depends on N only (CUDA-graph capturable) and the background work on the count.
 * A camera outside the ellipsoid sets the status word: MN_ERR_SPHERE is returned by the next mn_check_status, the results
 * of this call are then undefined.
 *   fg / bg: models of the same kind (use_cascade) and head (sh_deg); image_indices_d required iff either has an appearance
 *   embedding; sphere_radius3_d NULL = the unit sphere at the origin;
 *   include_xyz_real / cluster_2d as for mn_points_outside (render.py:304-305);
 *   z_steps_bg_d = torch.linspace(0,1,coarse_samples/2), u_fine_bg_d = torch.linspace(0,1,fine_samples/2), passed in like
 *   z_steps_d / u_fine_d (SURVEY §8c: these values are not a subset of the longer vectors).
 * mn_render_outputs: nullable device pointers named after the result keys of the final type (fine, coarse when
 * fine_samples == 0) and of the coarse type under use_cascade with fine_samples > 0; rgb is required.  fg_* / bg_* are the
 * two terms of the blend (get_bg_fg_rgb); bg_lambda* are computed either way. */
typedef struct mn_render_outputs {
    float* rgb;               /* [N,3] rgb_<final>                                   */
    float* depth;             /* [N]   depth_<final>                                 */
    float* depth_var;         /* [N]   depth_variance_<final> (foreground only)      */
    float* bg_lambda;         /* [N]   bg_lambda_<final>                             */
    float* fg_rgb;            /* [N,3] fg_rgb_<final>                                */
    float* bg_rgb;            /* [N,3] bg_rgb_<final>                                */
    float* fg_depth;          /* [N]   fg_depth_<final>                              */
    float* bg_depth;          /* [N]   bg_depth_<final>                              */
    float* rgb_coarse;        /* [N,3] rgb_coarse (use_cascade, fine_samples > 0)    */
    float* bg_lambda_coarse;  /* [N]   bg_lambda_coarse                              */
    float* fg_rgb_coarse;     /* [N,3] fg_rgb_coarse                                 */
    float* bg_rgb_coarse;     /* [N,3] bg_rgb_coarse                                 */
} mn_render_outputs;
size_t mn_render_rays_bg_workspace_bytes(const mn_model* fg, const mn_model* bg, int64_t N, int coarse_samples, int fine_samples,
                                         int use_cascade, int sh_deg, int precision);
int mn_render_rays_bg(mn_ctx* ctx, mn_model* fg, mn_model* bg, const float* rays_d, const float* image_indices_d, int64_t N,
                      const float* sphere_center3_d, const float* sphere_radius3_d, int include_xyz_real, int cluster_2d,
                      const float* z_steps_d, const float* z_steps_bg_d, int coarse_samples, const float* u_fine_d,
                      const float* u_fine_bg_d, int fine_samples, int use_cascade, int sh_deg, int precision,
                      const mn_render_outputs* out, void* workspace_d, size_t workspace_bytes, void* stream);

/* Fused per-ray all-gather over peer memory (SURVEY.md §8e): stores this rank's (rgb, depth) rows [row0, row0+n) into
 * every buffer of peer_bufs[0..n_peers) - HOST array of device pointers to [n_total, 4] fp32 buffers, one per rank,
 * peer-mapped into this process (e.g. torch symmetric memory) - with 16-byte P2P stores.  Cross-rank ordering (nobody
 * still reads the previous contents; everybody's stores have landed) is the caller's: a barrier before and after. */
int mn_peer_gather_store(mn_ctx* ctx, const float* rgb_d, const float* depth_d, int64_t n, int64_t row0,
                         const void* const* peer_bufs, int n_peers, void* stream);

/* ---- cluster masks ------------------------------------------- scripts/create_cluster_masks.py ----
 * The per-image hot loop of create_cluster_masks.py:155-201 (SURVEY.md §8f-3): for every ray, the minimum over
 * its S samples (z = near(1-t) + far t, t = z_steps_d [S] = torch.linspace(0,1,S) passed in) of
 * d(sample, centroid_k) / (min_j d(sample, centroid_j) + 1e-8), distances over (y,z) only iff cluster_2d.
 *   rays_d [N,8]; centroids_d [K,3];  ratios_out_d optional [N,K];
 *   mask_out_d optional uint8 [K,N] = (ratio <= boundary_margin), i.e. one [H,W] pixel mask per cluster
 *   (create_cluster_masks.py:199-201).  At least one output must be given. */
int mn_cluster_min_dist_ratios(mn_ctx* ctx, const float* rays_d, int64_t N, const float* z_steps_d, int S,
                               const float* centroids_d, int K, int cluster_2d, float boundary_margin,
                               float* ratios_out_d, unsigned char* mask_out_d, void* stream);

/* ---- training: gradients of the path ------------------------------------ SURVEY.md §8f-1 --------
 * What `loss.backward()` computes through the hot path in the reference's training step
 * (runner.py:346-378 -> :265).  Gradient flow is the reference's: per-sample (rgb, sigma) receive
 * gradients from the composited colour and from bg_lambda; resampling weights are detached
 * (rendering.py:215) and depth terms are computed under no_grad (rendering.py:381), so neither
 * contributes; sample positions carry no gradient.  fp32 (CUDA-core) arithmetic only in this ABI
 * version: the training forward always runs in MN_PREC_FP32.                                      */

/* d(sum(rgb * grad_rgb) + sum(bg_lambda * grad_lambda)) / d raw   for mn_composite's inputs
 * (rendering.py:336-373): same raw/z/raw2/z2/last_delta/flip as the forward call;
 *   grad_rgb_d [N,3]; grad_lambda_d optional [N];
 *   grad_raw_d [N,S,4] and (iff S2 > 0) grad_raw2_d [N,S2,4] receive d/d(r,g,b,sigma) per sample. */
int mn_composite_backward(mn_ctx* ctx, const float* raw_d, const float* z_d, int S, const float* raw2_d,
                          const float* z2_d, int S2, const float* last_delta_d, int64_t N, int flip,
                          const float* grad_rgb_d, const float* grad_lambda_d, float* grad_raw_d, float* grad_raw2_d,
                          void* stream);
/* Backward of mn_sh_to_rgb (spherical_harmonics.py:55-106 + sigmoid, rendering.py:301-306):
 *   grad_out_d [B,4] -> grad_coef_d [B, coef_stride] (all 3*(deg+1)^2 + 1 used columns written). */
int mn_sh_to_rgb_backward(mn_ctx* ctx, int deg, const float* coef_d, int64_t coef_stride, const float* dirs_d,
                          int64_t dir_stride, int dir_div, int64_t B, int apply_sigmoid, const float* grad_out_d,
                          float* grad_coef_d, void* stream);

/* Training forward of nn.Module.__call__ (nerf.py:115-160, cascade.py:13-18, mega_nerf.py:19-61): same
 * result as mn_model_forward(precision = MN_PREC_FP32, sigma_only = 0) and, in addition, everything the
 * backward pass needs (routing tables of this call, every layer's activations) is written to the
 * caller-owned `tape_d` (mn_model_tape_bytes(m, B) bytes), which must stay untouched until
 * mn_model_backward has consumed it.  workspace as for mn_model_forward(MN_PREC_FP32). */
size_t mn_model_tape_bytes(const mn_model* m, int64_t B);
int mn_model_forward_train(mn_ctx* ctx, mn_model* m, const mn_rows* rows, int64_t B, int use_coarse,
                           const float* sigma_noise_d, float* out_d, void* tape_d, size_t tape_bytes, void* workspace_d,
                           size_t workspace_bytes, void* stream);
/* Parameter gradients.  grad_out_d [B, rgb_dim+1] is dL/d(out) of the matching mn_model_forward_train
 * call (same B / use_coarse / tape).  Gradients are ACCUMULATED (+=) into param_grads_d, a caller-zeroed
 * fp32 block of mn_model_grad_floats(m) = n_sub * stride floats: sub-module s owns [s*stride, (s+1)*stride)
 * and inside it every tensor sits at the offset mn_model_param_offsets reports, in the reference's
 * state-dict layout (nn.Linear weight [out,in] row-major, embedding [count,dim]).
 * mn_model_param_offsets fills out[0..MN_PARAM_OFFSETS): stride, xyz_encodings.{0..15}.0.weight,
 * xyz_encodings.{0..15}.0.bias (-1 beyond `layers`), sigma.weight, sigma.bias, xyz_encoding_final.weight,
 * .bias, dir_a_encoding.0.weight, .bias, rgb.weight, .bias, embedding_a.weight, affine.weight, affine.bias. */
#define MN_PARAM_OFFSETS 44
size_t mn_model_backward_workspace_bytes(const mn_model* m, int64_t B);
int64_t mn_model_grad_floats(const mn_model* m);
int mn_model_param_offsets(const mn_model* m, int64_t* out, int n);
int mn_model_backward(mn_ctx* ctx, mn_model* m, int64_t B, int use_coarse, const float* grad_out_d, const void* tape_d,
                      size_t tape_bytes, float* param_grads_d, void* workspace_d, size_t workspace_bytes, void* stream);

/* ---- the same two passes on the tensor cores (precision tc_f16) --------------------------------------------------
 * What the reference does on a GPU: Linear layers in fp16 with fp32 accumulation under autocast, gradients scaled into
 * fp16 range (runner.py:243-274, opts.py:99).  Forward = the tc_f16 inference kernel writing every layer's fp16
 * activations to the tape; backward = data gradients on transposed fp16 weight images (ReLU masks from the tape, gradient
 * images scaled by a power of two chosen from max|grad_out|), weight gradients as wgmma contractions of the two tapes
 * over the slot axis, fp32 accumulation, fp32 atomics into param_grads_d.  Same argument meaning as the fp32 entry points
 * above; covers layer_dim 256, 512 (up to 10 trunk layers) and 768..2048 (a multiple of 256; the layer-GEMM path, backward
 * one tile group at a time) with a direction / appearance head and either rgb_dim 3 or a raw SH head (rgb_dim <= 80, i.e.
 * sh_deg <= 4; rgb_dim 48 and 75 run on the layer-GEMM path at 256 and 512 wide too), no affine appearance (mn_model_train_tc_supported), everything else returns MN_ERR_UNSUPPORTED - use the fp32 entry points.
 * The first recording call allocates the transposed weight images of the backward (about 4.25 MiB per 512-wide and 71 MB
 * per 2048-wide sub-module).
 * Gradients agree with the fp32 path to ~1e-2 of each tensor's scale (fp16 operands, like the reference under autocast);
 * the fp32 entry points remain the parity mode. */
int mn_model_train_tc_supported(const mn_model* m);
size_t mn_model_tape_bytes_tc(const mn_model* m, int64_t B);
int mn_model_forward_train_tc(mn_ctx* ctx, mn_model* m, const mn_rows* rows, int64_t B, int use_coarse,
                              const float* sigma_noise_d, float* out_d, void* tape_d, size_t tape_bytes, void* workspace_d,
                              size_t workspace_bytes, void* stream);
size_t mn_model_backward_workspace_bytes_tc(const mn_model* m, int64_t B);
int mn_model_backward_tc(mn_ctx* ctx, mn_model* m, int64_t B, int use_coarse, const float* grad_out_d, const void* tape_d,
                         size_t tape_bytes, float* param_grads_d, void* workspace_d, size_t workspace_bytes, void* stream);

/* ---- test hook (host only, no CUDA call) ---------------------------------------------------------------------------
 * The stage program of the tensor-core MLP kernel (csrc/mn_mlp_wg.cuh, precision tc_f16) for one network shape: `desc` as for
 * mn_model_create (only the per-sub-module fields matter).  The producer and both consumer warpgroups walk this program, one
 * entry per weight-ring stage of one 128-row tile.  table_out receives up to cap_entries entries of 8 unsigned ints: weight
 * byte offset in the sub-module's pack, weight bytes, B rows (N), K columns, first K column of the A operand, feature-segment
 * byte offset and bytes (first stage of a feature segment, else 0), flags | GEMM << 8 | N-chunk << 16 (flags: 1 A from the
 * feature buffer, 2 first / 4 last stage of a feature segment, 8 lo planes, 16 first / 32 last stage of an accumulator).
 * info[8] = {entries, entries of a sigma_only call, bytes of one weight plane of a sub-module, ring stages, shared-memory bytes,
 * feature-tile bytes, ring-stage bytes, K columns per stage}.  Returns MN_ERR_UNSUPPORTED for shapes only the fp32 kernels
 * run, MN_ERR_WORKSPACE when cap_entries is too small.  Used by tests/test_tp_program.py and tests/tp_protocol_sim.py. */
int mn_debug_tp_program(const mn_model_desc* desc, unsigned int* table_out, int cap_entries, int* info8);

#ifdef __cplusplus
}
#endif
#endif /* MN_B200_H */
