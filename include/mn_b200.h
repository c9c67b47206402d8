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
/* A weight repack that a CUDA graph can replay.  mn_model_bind_weights records the tensors of *w as the sources of sub-module
 * `sub` - they must stay allocated at the same addresses (a training step updates parameters in place) - and, once every
 * sub-module is bound, builds the model's table of re-layouts in device memory.  It allocates the fp16 forward images if they
 * do not exist yet, synchronises the device and uploads the table: a set-up call, not for a captured region.  The transposed
 * images of the tensor-core backward are covered iff they exist when the sub-module is bound - the first recording call on the
 * tensor cores allocates them; a network trained in fp32 never holds them.  Binding a sub-module again replaces its sources; a
 * table that a graph captured earlier may read is never freed before the model (an identical table is reused).
 * mn_model_repack then re-packs every image of every sub-module from the bound tensors - the fp32 layouts, the fp16 forward
 * images and the transposed data-gradient images - in two launches on `stream`, with no host upload and no allocation, the same
 * images mn_model_set_weights writes from the same values.  MN_ERR_INVALID until every sub-module is bound, and if the
 * transposed images were allocated after a sub-module was bound (bind it again). */
int mn_model_bind_weights(mn_model* m, int sub, const mn_nerf_weights* w);
int mn_model_repack(mn_ctx* ctx, mn_model* m, void* stream);

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
/* ---- expert-parallel ("one centroid per GPU") query --------------------------- models/mega_nerf.py:19-61 ----
 * MegaNeRF.forward with sub-module k evaluated on rank k mod world only (mega_nerf_b200/expert_parallel.py).  Three device
 * steps around two equal-split all-to-alls, none of which synchronises the host or takes a size from the device:
 *   home:  mn_model_route -> mn_model_ep_dispatch -> [send segments, counts]
 *   owner: mn_model_forward_assigned on the received segments -> [results]
 *   home:  mn_model_ep_combine on the returned segments.
 * Every rank must pass the same capacity row count B_cap >= B: the segments are sized from it.  B_cap == B on every rank is
 * the plain case; a query whose row count differs from rank to rank (the rays that reach a background network) passes the
 * maximum over the ranks.
 *
 * Rows of one segment: B_cap x max_multiplicity (mn_model_set_max_multiplicity; 1 under hard routing), the router's own slot
 * bound, so the pairs of one query fit any one segment.  A row within the margin of more sub-modules than max_multiplicity
 * can push a segment past it; its result is then NaN and MN_ERR_WORKSPACE follows at the next mn_check_status. */
int64_t mn_model_ep_segment_rows(const mn_model* m, int64_t B);
/* Dispatch (mega_nerf.py:19-61, the `cluster_mask` selection of every sub-module): the (row, sub-module) pairs of
 * x_d [B, cols] (the model's rows; the first 3 columns are routing-only with xyz_real) from the router's output - assign_d
 * int32 [B] (boundary_margin == 1) or weights_d [B, n_sub] (> 1, pairs where the weight is > 0) - ordered by destination
 * rank (k mod world), sub-module, row.  Pair p for destination d occupies row d * S + p (S = mn_model_ep_segment_rows(m, B_cap))
 * of:
 *   send_d [world * S, c + 1 (+1)]: the child's input (cols - 3 with xyz_real, else cols columns), the sub-module id as a
 *     float and, if sigma_noise_d [B] is given, the row's density noise; rows past a segment's pairs carry id -1;
 *   pair_row_d int32 [world * S] (home row, -1 past the pairs) and pair_w_d [world * S] (blend weight; margin > 1 only).
 * counts_d int32 [world, n_sub]: pairs per (destination, sub-module).  row_slots_d int32: [B] the slot of each row's pair
 * (hard routing) or [B, n_sub] the slot per sub-module, -1 where none (margin > 1) - what mn_model_ep_combine reads.
 * B is this rank's own row count: the rows routed, counted and scattered (routing still follows B, cdist's direct path for
 * B <= 25 included).  B == 0 with B_cap > 0 still writes the segments: id -1 in every payload row, pair_row -1, pair_w 0 and
 * counts 0; x_d, assign_d / weights_d and row_slots_d may then be NULL, but sigma_noise_d must be non-NULL iff the payload
 * rows carry the noise column (it sets the row width; nothing is read from it). */
size_t mn_model_ep_dispatch_workspace_bytes(const mn_model* m, int64_t B, int world);
int mn_model_ep_dispatch(mn_ctx* ctx, mn_model* m, const float* x_d, int64_t B, int64_t B_cap, int cols, const int32_t* assign_d,
                         const float* weights_d, const float* sigma_noise_d, int world, float* send_d, int32_t* counts_d,
                         int32_t* pair_row_d, float* pair_w_d, int32_t* row_slots_d, void* workspace_d, size_t workspace_bytes,
                         void* stream);
/* Owner call (mega_nerf.py:19-61, `sub_module(x[cluster_mask])` of the sub-modules this rank owns): rows_d [n, cols + 1 (+1)]
 * in the layout mn_model_ep_dispatch sends - the child's input (cols columns), the sub-module id, the density noise iff
 * has_noise - each row through its own sub-module, all in one call; rows with id -1 are skipped (their out_d rows are not
 * written).  out_d [n, rgb_dim + 1].  Only the weights of the sub-modules that occur need to be set. */
size_t mn_model_forward_assigned_workspace_bytes(const mn_model* m, int64_t n, int precision);
int mn_model_forward_assigned(mn_ctx* ctx, mn_model* m, const float* rows_d, int64_t n, int cols, int has_noise, int precision,
                              float* out_d, void* workspace_d, size_t workspace_bytes, void* stream);
/* Combine (mega_nerf.py:34,46-49): out_d [B, rgb_dim + 1] from back_d [world * S, rgb_dim + 1] (the owners' results in
 * the dispatch's slots): every row starts from 0 and adds back x w over its pairs in ascending sub-module order, multiply
 * and add rounded separately as `results[mask] += sub_result * weights[mask, i]`; hard routing copies the row's result.
 * row_slots_d / pair_w_d as written by mn_model_ep_dispatch. */
int mn_model_ep_combine(mn_ctx* ctx, mn_model* m, int64_t B, const int32_t* row_slots_d, const float* pair_w_d, const float* back_d,
                        float* out_d, void* stream);
/* Training under expert parallelism: the same three steps recording, then their backward in reverse, around the same
 * equal-split all-to-alls (the result gradients travel home -> owner like the rows).
 *   home:  mn_model_ep_combine_backward: dback_d [n_slots, rgb_dim + 1] (n_slots = world * S) from dout_d [B, rgb_dim + 1],
 *          the gradient of mn_model_ep_combine's output: slot s gets w[s] x dout[pair_row[s]] (one fp32 multiply; hard routing
 *          copies dout[pair_row[s]]), 0 where pair_row[s] is -1.  pair_row_d / pair_w_d as written by mn_model_ep_dispatch.
 *   owner: mn_model_forward_assigned_train, then mn_model_backward_assigned on the returned result gradients.
 * The owner's tape is sized by max_pairs, the pairs that actually arrived (the sum of the received counts: one host read per
 * query), not by the n = world * S padded rows: mn_model_assigned_tape_bytes(m, max_pairs, precision).  The rows stay where
 * they arrived.  More pairs than max_pairs cannot write past the tape: the extra pairs are dropped, their out_d rows are NaN
 * and MN_ERR_WORKSPACE follows at the next mn_check_status.
 * mn_model_forward_assigned_train: mn_model_forward_assigned that also writes the tape; precision MN_PREC_FP32 (the fp32 kernels
 * of mn_model_forward_train) or MN_PREC_TC_F16 (those of mn_model_forward_train_tc, same coverage); out_d rows with id -1 are NaN.
 * mn_model_backward_assigned: grad_out_d [n, rgb_dim + 1] is dL/d(out) of the matching recording call (same n, max_pairs,
 * precision, tape); parameter gradients are ACCUMULATED into param_grads_d as by mn_model_backward (only the sub-modules that
 * occur in the rows get non-zero entries). */
int mn_model_ep_combine_backward(mn_ctx* ctx, mn_model* m, int64_t n_slots, const int32_t* pair_row_d, const float* pair_w_d,
                                 const float* dout_d, float* dback_d, void* stream);
size_t mn_model_assigned_tape_bytes(const mn_model* m, int64_t max_pairs, int precision);
size_t mn_model_forward_assigned_train_workspace_bytes(const mn_model* m, int64_t n);
int mn_model_forward_assigned_train(mn_ctx* ctx, mn_model* m, const float* rows_d, int64_t n, int cols, int has_noise, int64_t max_pairs,
                                    int precision, float* out_d, void* tape_d, size_t tape_bytes, void* workspace_d, size_t workspace_bytes,
                                    void* stream);
size_t mn_model_backward_assigned_workspace_bytes(const mn_model* m, int64_t max_pairs, int precision);
int mn_model_backward_assigned(mn_ctx* ctx, mn_model* m, int64_t n, int64_t max_pairs, int precision, const float* grad_out_d,
                               const void* tape_d, size_t tape_bytes, float* param_grads_d, void* workspace_d, size_t workspace_bytes,
                               void* stream);
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

/* ---- the same through an occupancy grid (an approximate render mode the caller opts into) --------------------------------
 * mn_render_rays / mn_render_rays_bg, except that the foreground samples of both passes (coarse and fine) that lie in a cell the
 * grid marks empty are not queried: their raw row [rgb, sigma] (after the SH head, for one) is exactly (0, 0, 0, 0), and every
 * later stage - composite, resampling, merge, background pass, blend - runs unchanged on it.  The background pass is never
 * masked.  For a sample point x, per axis a: u_a = x_a * scale_a + offset_a (two separately rounded fp32 operations, no FMA),
 * i_a = (int)floorf(u_a * reso); the sample is skipped iff 0 <= u_a < 1 on all three axes and bit (i_0 * reso + i_1) * reso + i_2
 * (bit c & 31 of bits[c >> 5]) is 0 - so a point outside the box, or a NaN point, is always queried.  The bit order is the
 * lattice order of mn_model_density_grid with the same offset / scale (the octree's tree.offset / tree.invradius).  With every
 * bit set the results equal those of mn_render_rays(_bg).
 * The queried samples are compacted on the device in ascending order and their count stays there: no host sync, the launch
 * sequence depends on N only (CUDA-graph capturable).  counts_out_d: NULL, or int32 [2] receiving the queried foreground rows of
 * the coarse [0] and of the fine [1] pass (the latter written only with fine_samples > 0).  N * max(coarse, fine-query samples)
 * must stay below 2^31; reso 1 .. MN_OCC_MAX_RESO.  The grid is read during the call only. */
#define MN_OCC_MAX_RESO 2048
typedef struct mn_occupancy {
    const uint32_t* bits;     /* device, ceil(reso^3 / 32) words                     */
    int reso;
    float offset[3];
    float scale[3];
} mn_occupancy;
size_t mn_render_rays_occ_workspace_bytes(const mn_model* m, int64_t N, int coarse_samples, int fine_samples, int use_cascade,
                                          int sh_deg, int precision);
int mn_render_rays_occ(mn_ctx* ctx, mn_model* m, const float* rays_d, const float* image_indices_d, int64_t N,
                       const float* z_steps_d, int coarse_samples, const float* u_fine_d, int fine_samples, int use_cascade,
                       int sh_deg, int precision, const mn_occupancy* occ, int32_t* counts_out_d, float* rgb_out_d,
                       float* depth_out_d, float* depth_var_out_d, float* rgb_coarse_out_d, void* workspace_d,
                       size_t workspace_bytes, void* stream);
size_t mn_render_rays_bg_occ_workspace_bytes(const mn_model* fg, const mn_model* bg, int64_t N, int coarse_samples, int fine_samples,
                                             int use_cascade, int sh_deg, int precision);
int mn_render_rays_bg_occ(mn_ctx* ctx, mn_model* fg, mn_model* bg, const float* rays_d, const float* image_indices_d, int64_t N,
                          const float* sphere_center3_d, const float* sphere_radius3_d, int include_xyz_real, int cluster_2d,
                          const float* z_steps_d, const float* z_steps_bg_d, int coarse_samples, const float* u_fine_d,
                          const float* u_fine_bg_d, int fine_samples, int use_cascade, int sh_deg, int precision,
                          const mn_occupancy* occ, int32_t* counts_out_d, const mn_render_outputs* out, void* workspace_d,
                          size_t workspace_bytes, void* stream);

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
 * above; covers layer_dim 256..4096 with 2..16 trunk layers (256 and 512 wide up to 12 layers on the fused kernel; every other
 * width and depth on the layer-GEMM path, backward one tile group at a time) with a direction / appearance head and either rgb_dim 3 or a raw SH head (rgb_dim <= 80, i.e.
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

/* ---- the recording foreground render in one call ------------------------- mega_nerf/rendering.py:15-248, train mode ----
 * render_rays(nerf, bg_nerf=None, ...) while training (runner.py:347-358): the stage entry points of the training path in their
 * order - coarse depths with jitter, recording coarse query (+ SH head), the cascade's coarse colour, the weights of the
 * detached coarse composite, inverse-CDF resampling, sort_cat under use_cascade, recording fine query, merge + volume
 * rendering - sequenced on `stream` with no allocation and no host sync, the same results as those calls.  Every random input
 * is the caller's, drawn as the reference draws it:
 *   jitter_d [N, coarse_samples] (torch.rand; NULL iff perturb == 0); sigma_noise_coarse_d [N * coarse_samples] and
 *   sigma_noise_fine_d [N * Sq] (Sq = fine_samples, or coarse_samples + fine_samples under use_cascade; NULL: no noise);
 *   u_fine_d [N, fine_samples] (torch.rand, or the rows of torch.linspace(0, 1, fine_samples) when perturb == 0).
 * fine_samples > 0; z_steps_d, use_cascade, sh_deg and image_indices_d as for mn_render_rays.  precision MN_PREC_FP32 (the
 * kernels of mn_model_forward_train) or MN_PREC_TC_F16 (those of mn_model_forward_train_tc, same coverage and errors).
 * Outputs: rgb_out_d [N,3] rgb_fine; depth_out_d / depth_var_out_d optional [N]; rgb_coarse_out_d [N,3], required under
 * use_cascade.  tape_d (mn_render_rays_train_tape_bytes) receives what the backward needs - the composite inputs and both model
 * tapes - and must stay untouched until mn_render_rays_train_backward has consumed it; its layout depends on (N, coarse_samples,
 * fine_samples, use_cascade, sh_deg, precision) and the model only.  workspace_d: mn_render_rays_train_workspace_bytes.
 * mn_render_rays_train_backward (same N, sample counts, flags, precision and tape): grad_rgb_d [N,3] = dL/d rgb_fine and, under
 * use_cascade, grad_rgb_coarse_d [N,3] = dL/d rgb_coarse (NULL: no gradient, the coarse query's backward is skipped); runs the
 * composite backward(s), then the fine and the coarse model backward, and ACCUMULATES the parameter gradients into
 * param_grads_d as mn_model_backward does (mn_model_grad_floats, mn_model_param_offsets).  No host sync. */
size_t mn_render_rays_train_tape_bytes(const mn_model* m, int64_t N, int coarse_samples, int fine_samples, int use_cascade,
                                       int sh_deg, int precision);
size_t mn_render_rays_train_workspace_bytes(const mn_model* m, int64_t N, int coarse_samples, int fine_samples, int use_cascade,
                                            int sh_deg, int precision);
int mn_render_rays_train(mn_ctx* ctx, mn_model* m, const float* rays_d, const float* image_indices_d, int64_t N,
                         const float* z_steps_d, const float* jitter_d, float perturb, int coarse_samples,
                         const float* sigma_noise_coarse_d, const float* u_fine_d, const float* sigma_noise_fine_d, int fine_samples,
                         int use_cascade, int sh_deg, int precision, float* rgb_out_d, float* depth_out_d, float* depth_var_out_d,
                         float* rgb_coarse_out_d, void* tape_d, size_t tape_bytes, void* workspace_d, size_t workspace_bytes,
                         void* stream);
size_t mn_render_rays_train_backward_workspace_bytes(const mn_model* m, int64_t N, int coarse_samples, int fine_samples,
                                                     int use_cascade, int sh_deg, int precision);
int mn_render_rays_train_backward(mn_ctx* ctx, mn_model* m, int64_t N, int coarse_samples, int fine_samples, int use_cascade,
                                  int sh_deg, int precision, const float* grad_rgb_d, const float* grad_rgb_coarse_d,
                                  const void* tape_d, size_t tape_bytes, float* param_grads_d, void* workspace_d,
                                  size_t workspace_bytes, void* stream);

/* mn_render_rays_train_bg: the recording render of render_rays(nerf, bg_nerf, ...) in train mode (rendering.py:34-75,
 * render.py `_render`) as ONE call: the device sphere split and stable compaction of mn_render_rays_bg, the background network's
 * two-pass recording render over the compacted rays (their count stays on the device: every stage, the router, the encoders and
 * the MLP tiles stop at it), the foreground's recording render with the far override, last delta and bg_lambda, then the lambda
 * blend rgb = fg + bg_lambda * bg of the final type and, under use_cascade, of the coarse one.  No allocation, no host sync, a
 * static launch sequence (CUDA-graph capturable); with no background ray the background kernels launch and do nothing.
 *   fg / bg, image_indices_d, sphere_center3_d / sphere_radius3_d, include_xyz_real, cluster_2d, z_steps_d / z_steps_bg_d: as for
 *   mn_render_rays_bg; precision / bg_precision: each network's training precision (MN_PREC_FP32 or MN_PREC_TC_F16);
 *   foreground draws as for mn_render_rays_train; background draws jitter_bg_d [rows, coarse_samples/2] (NULL iff perturb == 0),
 *   sigma_noise_coarse_bg_d [rows * coarse_samples/2], u_fine_bg_d [rows, fine_samples/2], sigma_noise_fine_bg_d
 *   [rows * Sq_bg] (Sq_bg = fine_samples/2, or coarse_samples/2 + fine_samples/2 under use_cascade).  bg_draws_by_ray = 0: row p
 *   of each block belongs to the p-th background ray in ascending ray order (rows = the background count, render_rays' stream);
 *   1: row i belongs to ray i (rows = N), rows of rays that stay in the foreground are not read.
 *   out: as for mn_render_rays_bg; rgb, bg_lambda required, and rgb_coarse and bg_lambda_coarse under use_cascade.
 * A camera outside the ellipsoid sets the status word (MN_ERR_SPHERE at the next mn_check_status).  tape_d
 * (mn_render_rays_train_bg_tape_bytes) must stay untouched until mn_render_rays_train_bg_backward has consumed it.
 * mn_render_rays_train_bg_backward (same sizes, flags, precisions and tape): grad_rgb_d [N,3] = dL/d rgb_fine, grad_rgb_coarse_d
 * as for mn_render_rays_train_backward; runs the blend backward, the foreground composite backward (its bg_lambda included) and
 * model backwards, then the background composite and model backwards over the device count, and ACCUMULATES into
 * param_grads_d (foreground) and bg_param_grads_d (background) as mn_model_backward does.  No host sync. */
size_t mn_render_rays_train_bg_tape_bytes(const mn_model* fg, const mn_model* bg, int64_t N, int coarse_samples, int fine_samples,
                                          int use_cascade, int sh_deg, int precision, int bg_precision);
size_t mn_render_rays_train_bg_workspace_bytes(const mn_model* fg, const mn_model* bg, int64_t N, int coarse_samples, int fine_samples,
                                               int use_cascade, int sh_deg, int precision, int bg_precision);
int mn_render_rays_train_bg(mn_ctx* ctx, mn_model* fg, mn_model* bg, const float* rays_d, const float* image_indices_d, int64_t N,
                            const float* sphere_center3_d, const float* sphere_radius3_d, int include_xyz_real, int cluster_2d,
                            const float* z_steps_d, const float* z_steps_bg_d, const float* jitter_d, const float* jitter_bg_d,
                            float perturb, int coarse_samples, const float* sigma_noise_coarse_d, const float* sigma_noise_coarse_bg_d,
                            const float* u_fine_d, const float* u_fine_bg_d, const float* sigma_noise_fine_d,
                            const float* sigma_noise_fine_bg_d, int fine_samples, int use_cascade, int sh_deg, int precision,
                            int bg_precision, int bg_draws_by_ray, const mn_render_outputs* out, void* tape_d, size_t tape_bytes,
                            void* workspace_d, size_t workspace_bytes, void* stream);
size_t mn_render_rays_train_bg_backward_workspace_bytes(const mn_model* fg, const mn_model* bg, int64_t N, int coarse_samples,
                                                        int fine_samples, int use_cascade, int sh_deg, int precision, int bg_precision);
int mn_render_rays_train_bg_backward(mn_ctx* ctx, mn_model* fg, mn_model* bg, int64_t N, int coarse_samples, int fine_samples,
                                     int use_cascade, int sh_deg, int precision, int bg_precision, const float* grad_rgb_d,
                                     const float* grad_rgb_coarse_d, const void* tape_d, size_t tape_bytes, float* param_grads_d,
                                     float* bg_param_grads_d, void* workspace_d, size_t workspace_bytes, void* stream);

/* ---- the training renders through an occupancy grid (an approximate training mode the caller opts into) -------------------
 * mn_render_rays_train / mn_render_rays_train_bg, except that the foreground samples of both passes that the grid skips (the
 * grid, the cell test and the frame of mn_render_rays_occ) are not queried: their raw row [rgb, sigma] (after the SH head, for
 * one) is exactly (0, 0, 0, 0), and every later stage - the coarse composite and the resampling weights, the fine draws (tested
 * and skipped the same way), the merge, the final composite, the background pass (never masked) and the blend - runs unchanged on
 * it.  A skipped sample reaches no parameter: the backward runs the composite backward(s) over every sample, then the SH head's
 * and the model's backward over the queried rows only, so every gradient equals that of the stage path with the skipped raw rows
 * replaced by zero.  The random inputs are those of the unmasked call, drawn for every sample (density noise [N * S] in sample
 * order); a queried sample uses its own draw.  With every bit set the results equal those of mn_render_rays_train(_bg).
 * The queried samples are compacted on the device and their count stays there: no host sync, the launch sequence depends on N
 * only (CUDA-graph capturable).  counts_out_d: NULL, or int32 [2] receiving the queried foreground rows of the coarse [0] and the
 * fine [1] pass.  N * max(coarse_samples, Sq) must stay below 2^31; reso 1 .. MN_OCC_MAX_RESO.  The grid is read during the
 * forward call only.  The tape also holds each pass's compacted sample indices and counts, so the size queries and the backward
 * take the unmasked call's arguments and need no grid; a tape written by an _occ call is consumed by the _occ backward only. */
size_t mn_render_rays_train_occ_tape_bytes(const mn_model* m, int64_t N, int coarse_samples, int fine_samples, int use_cascade,
                                           int sh_deg, int precision);
size_t mn_render_rays_train_occ_workspace_bytes(const mn_model* m, int64_t N, int coarse_samples, int fine_samples, int use_cascade,
                                                int sh_deg, int precision);
int mn_render_rays_train_occ(mn_ctx* ctx, mn_model* m, const float* rays_d, const float* image_indices_d, int64_t N,
                             const float* z_steps_d, const float* jitter_d, float perturb, int coarse_samples,
                             const float* sigma_noise_coarse_d, const float* u_fine_d, const float* sigma_noise_fine_d, int fine_samples,
                             int use_cascade, int sh_deg, int precision, const mn_occupancy* occ, int32_t* counts_out_d, float* rgb_out_d,
                             float* depth_out_d, float* depth_var_out_d, float* rgb_coarse_out_d, void* tape_d, size_t tape_bytes,
                             void* workspace_d, size_t workspace_bytes, void* stream);
size_t mn_render_rays_train_occ_backward_workspace_bytes(const mn_model* m, int64_t N, int coarse_samples, int fine_samples,
                                                         int use_cascade, int sh_deg, int precision);
int mn_render_rays_train_occ_backward(mn_ctx* ctx, mn_model* m, int64_t N, int coarse_samples, int fine_samples, int use_cascade,
                                      int sh_deg, int precision, const float* grad_rgb_d, const float* grad_rgb_coarse_d,
                                      const void* tape_d, size_t tape_bytes, float* param_grads_d, void* workspace_d,
                                      size_t workspace_bytes, void* stream);
size_t mn_render_rays_train_bg_occ_tape_bytes(const mn_model* fg, const mn_model* bg, int64_t N, int coarse_samples, int fine_samples,
                                              int use_cascade, int sh_deg, int precision, int bg_precision);
size_t mn_render_rays_train_bg_occ_workspace_bytes(const mn_model* fg, const mn_model* bg, int64_t N, int coarse_samples,
                                                   int fine_samples, int use_cascade, int sh_deg, int precision, int bg_precision);
int mn_render_rays_train_bg_occ(mn_ctx* ctx, mn_model* fg, mn_model* bg, const float* rays_d, const float* image_indices_d, int64_t N,
                                const float* sphere_center3_d, const float* sphere_radius3_d, int include_xyz_real, int cluster_2d,
                                const float* z_steps_d, const float* z_steps_bg_d, const float* jitter_d, const float* jitter_bg_d,
                                float perturb, int coarse_samples, const float* sigma_noise_coarse_d,
                                const float* sigma_noise_coarse_bg_d, const float* u_fine_d, const float* u_fine_bg_d,
                                const float* sigma_noise_fine_d, const float* sigma_noise_fine_bg_d, int fine_samples, int use_cascade,
                                int sh_deg, int precision, int bg_precision, const mn_occupancy* occ, int32_t* counts_out_d,
                                int bg_draws_by_ray, const mn_render_outputs* out, void* tape_d, size_t tape_bytes, void* workspace_d,
                                size_t workspace_bytes, void* stream);
size_t mn_render_rays_train_bg_occ_backward_workspace_bytes(const mn_model* fg, const mn_model* bg, int64_t N, int coarse_samples,
                                                            int fine_samples, int use_cascade, int sh_deg, int precision,
                                                            int bg_precision);
int mn_render_rays_train_bg_occ_backward(mn_ctx* ctx, mn_model* fg, mn_model* bg, int64_t N, int coarse_samples, int fine_samples,
                                         int use_cascade, int sh_deg, int precision, int bg_precision, const float* grad_rgb_d,
                                         const float* grad_rgb_coarse_d, const void* tape_d, size_t tape_bytes, float* param_grads_d,
                                         float* bg_param_grads_d, void* workspace_d, size_t workspace_bytes, void* stream);

/* mn_occupancy_pack: bits_d [ceil(n / 32)] = the occupancy words of n cells, cell c occupied iff sigmas_d[c] >= thresh (a NaN sigma
 * gives an empty cell), in mn_occupancy's layout (bit c & 31 of word c >> 5; the bits past n are 0).  One warp ballot per word, no
 * atomics, no host sync: refreshes a grid in place, e.g. from mn_model_density_grid's sigmas, between replays of a captured graph
 * that reads it. */
int mn_occupancy_pack(mn_ctx* ctx, const float* sigmas_d, int64_t n, float thresh, uint32_t* bits_d, void* stream);

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
/* The same for one launch of the kernel: MN_TP_INFER is mn_debug_tp_program; MN_TP_TRAIN_FWD the recording forward of tc_f16
 * training (the forward program in the training variant's shared-memory layout); MN_TP_DGRAD the data-gradient chain of its
 * backward (one GEMM per Linear from dir_a_encoding down to trunk layer 1 on the transposed weight images, no feature segments;
 * info[1] == info[0], as no sigma_only form exists).  The training modes return MN_ERR_UNSUPPORTED unless the fused kernel
 * trains the shape (mn_model_train_tc_supported, and not the layer-GEMM engine).  Used by tests/test_tp_deep_train_program.py. */
#define MN_TP_INFER 0
#define MN_TP_TRAIN_FWD 1
#define MN_TP_DGRAD 2
int mn_debug_tp_program_mode(const mn_model_desc* desc, int mode, unsigned int* table_out, int cap_entries, int* info8);

/* ---- test hook (host only, no CUDA call): where the tensor-core training passes keep their intermediates -----------------
 * For a call of mn_model_forward_train_tc / mn_model_backward_tc over B rows of model m, out[] receives (indices MN_TCL_*):
 * the engine that runs the network's tensor-core forward (0 none, 1 the fused kernel, 2 the layer-GEMM engine); the tile count and byte size of
 * the tape and the byte offsets of its regions (routing counters, slot_row and slot_w or -1, encoder tiles, activation
 * records, fp32 head blocks); the bytes of one encoder tile and of one activation record; the padded widths of the encoder
 * segments and of the H / G images; the rows of the fp32 head block (sigma pre-activation, rgb, image id) and of the
 * head-gradient block; the backward workspace's size and the byte offsets, from workspace_d rounded up to 256 bytes, of the
 * gradient images (fused engine: one record per tile, laid out as the activation records), the head-gradient blocks, the
 * per-image embedding sums ([n_sub][app_count][emb_k] floats) and the scale S, then emb_k and the tiles the head-gradient
 * blocks cover; on the layer engine the offsets of the dZ_G image and of the two ping-pong gradient images of the last tile
 * group (-1 on the fused engine); the number of images of a record (layers + 2, or the trunk layers alone without
 * dir_a_encoding); whether tensor-core training covers the network (mn_model_train_tc_supported once packed); then per image
 * (trunk layers, F, G), its byte offset in the record and its columns.  Every tile image is [cols/8][128 rows][8] fp16.  Returns the entries written, or
 * MN_ERR_WORKSPACE when cap is too small.  The backward entries only mean something for networks trained on the tensor cores.
 * Used by tests/test_gpu_zzc_train_tc_stages.py and tests/test_gpu_zzd_infer_tc.py. */
#define MN_TCL_ENGINE 0
#define MN_TCL_N_TILES 1
#define MN_TCL_TAPE_BYTES 2
#define MN_TCL_TAPE_COUNTERS 3
#define MN_TCL_TAPE_SLOT_ROW 4
#define MN_TCL_TAPE_SLOT_W 5
#define MN_TCL_TAPE_XREG 6
#define MN_TCL_TAPE_ACT 7
#define MN_TCL_TAPE_F32 8
#define MN_TCL_X_TILE 9
#define MN_TCL_ACT_TILE 10
#define MN_TCL_KPE 11
#define MN_TCL_KAUX 12
#define MN_TCL_HC 13
#define MN_TCL_GC 14
#define MN_TCL_F32_SIGMA 15
#define MN_TCL_F32_RGB 16
#define MN_TCL_F32_ID 17
#define MN_TCL_F32_ROWS 18
#define MN_TCL_G32_SIGMA 19
#define MN_TCL_G32_RGB 20
#define MN_TCL_G32_ROWS 21
#define MN_TCL_BWD_BYTES 22
#define MN_TCL_BWD_DZ 23
#define MN_TCL_BWD_GF32 24
#define MN_TCL_BWD_EMB 25
#define MN_TCL_BWD_SCALE 26
#define MN_TCL_BWD_EMB_K 27
#define MN_TCL_BWD_HEAD_TILES 28
#define MN_TCL_BWD_DZG 29
#define MN_TCL_BWD_PP0 30
#define MN_TCL_BWD_PP1 31
#define MN_TCL_N_IMG 32
#define MN_TCL_TRAIN 33
#define MN_TCL_IMG 34
int mn_debug_tc_train_layout(const mn_model* m, int64_t B, int64_t* out, int cap);

/* ---- test hook (host only, no CUDA call): where the fp32 training passes keep their intermediates ------------------------
 * For a call of mn_model_forward_train / mn_model_backward over B rows of model m, out[] receives (indices MN_F32L_*): the
 * slots per tape tile TM and the number of TM-slot tiles; the tiles one CTA of the weight-gradient pass sums before its fp32
 * atomics; the tape's byte size and the byte offsets of its regions (routing counters, slot_row and slot_w or -1, the
 * activation tape); the backward workspace's size and the byte offset of the gradient tape inside it; then the first channel
 * of every activation-tape block (PE, aux = direction PE | embedding, trunk h_0.., F, G, rgb head output, affine Linear
 * output, sigma pre-activation, image id) and the channels per slot, and the same for the gradient tape (dZ of every trunk
 * layer, of F, of G, of the rgb Linear output, of the sigma pre-activation).  Channel c of slot r of tile t lies at float
 * (t * total + c) * TM + r of its tape.  Returns MN_F32L_COUNT, or MN_ERR_WORKSPACE when cap is too small.
 * Used by tests/test_gpu_zze_train_fp32_stages.py. */
#define MN_F32L_TM 0
#define MN_F32L_N_TILES 1
#define MN_F32L_CHUNK_TILES 2
#define MN_F32L_TAPE_BYTES 3
#define MN_F32L_TAPE_COUNTERS 4
#define MN_F32L_TAPE_SLOT_ROW 5
#define MN_F32L_TAPE_SLOT_W 6
#define MN_F32L_TAPE_ACT 7
#define MN_F32L_BWD_BYTES 8
#define MN_F32L_BWD_GRAD 9
#define MN_F32L_A_PE 10
#define MN_F32L_A_AUX 11
#define MN_F32L_A_H 12
#define MN_F32L_A_F 13
#define MN_F32L_A_G 14
#define MN_F32L_A_RGB 15
#define MN_F32L_A_LIN 16
#define MN_F32L_A_SIG 17
#define MN_F32L_A_ID 18
#define MN_F32L_A_TOTAL 19
#define MN_F32L_G_Z 20
#define MN_F32L_G_FINAL 21
#define MN_F32L_G_DIRA 22
#define MN_F32L_G_RGB 23
#define MN_F32L_G_SIG 24
#define MN_F32L_G_TOTAL 25
#define MN_F32L_COUNT 26
int mn_debug_fp32_train_layout(const mn_model* m, int64_t B, int64_t* out, int cap);

/* ---- test hook: the recording forward of any network the tensor cores run --------------------------------------------
 * mn_model_forward_train_tc's forward (arguments and tape as there, laid out as mn_debug_tc_train_layout reports) for every
 * network whose tc_f16 inference runs on the tensor cores, including the shapes tensor-core training does not cover (64..192
 * wide, affine appearance, no direction / appearance head).  Same plan, packed weights, encoder, GEMM order and epilogue
 * arithmetic as the tc_f16 inference call, so out_d equals that call's output; the tape holds what the forward computed on the
 * way.  Allocates no backward images.  MN_ERR_UNSUPPORTED for networks only the fp32 kernels run.  Used by
 * tests/test_gpu_zzd_infer_tc.py. */
int mn_debug_tc_forward_record(mn_ctx* ctx, mn_model* m, const mn_rows* rows, int64_t B, int use_coarse, const float* sigma_noise_d,
                               float* out_d, void* tape_d, size_t tape_bytes, void* workspace_d, size_t workspace_bytes, void* stream);

/* ---- test hook: the packed weight images of a model ------------------------------------------------------------------
 * which: 0 the fp32 forward layout of every sub-module (n_sub x PackedLayout floats), 1 the fp32 data-gradient layout
 * (n_sub x BwdLayout floats), 2 the fp16 hi / lo tensor-core forward images (n_sub x the plan's per-sub-module bytes), 3 the
 * transposed tensor-core data-gradient images (allocated by the first recording call on the tensor cores).  Returns the
 * image's byte size, 0 if it is not allocated (or `which` is out of range); with dst, copies min(size, cap) bytes device to
 * device on `stream` (0 and mn_last_error set if the copy fails).  Every image is zeroed when it is allocated and packs write
 * the same bytes from the same values, padding included, so two packs of equal weights are byte-identical.  Used by
 * tests/test_gpu_zzg_train_graph_shapes.py. */
size_t mn_debug_weight_images(const mn_model* m, int which, void* dst, size_t cap, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MN_B200_H */
