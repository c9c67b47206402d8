// Internal model representation shared by the packer, the router and the MLP kernels.
#pragma once
#include "mn_common.cuh"

#define MN_MAX_LAYERS 16
#define MN_MAX_SUB 64
#define MN_TILE 128     // rows of one tensor-core MLP tile
#define MN_BUCKET 512   // alignment of each sub-module's slot range (a multiple of MN_TILE: no tile mixes sub-modules); sets workspace and tape sizes

// Offsets (in floats) of each packed tensor inside one sub-module's fp32 buffer.  All matrices are
// stored K-major ("transposed": Wt[k][n] = W[n][k]) so that consecutive output channels are contiguous.
struct PackedLayout {
    int w[MN_MAX_LAYERS], b[MN_MAX_LAYERS], kin[MN_MAX_LAYERS];
    int sigma_w, sigma_b, final_w, final_b, dira_w, dira_b, rgb_w, rgb_b, emb, aff_w, aff_b;
    int total;
};

struct NetDims {
    int layers, L, in_xyz, in_dir, app, aux, rgb_dim, rgb_in, xyz_dim, nf_xyz, nf_dir, has_dir_a, affine,
        softplus, skip_mask, app_count, app_in_dira;
};

// ------------------------------------------------------------------------------------------------
// Training tapes (SURVEY.md §8f-1).  Both are tiled like the fp32 MLP kernel: tile t holds TM slots
// (TM = mn_tape_tm(L)), channel-major, i.e. value (channel c, slot r of tile t) lives at
// base[(t * C + c) * TM + r].  The ACTIVATION tape is written by the forward pass in training mode,
// the GRADIENT tape (dL/d pre-activation of every Linear) by the data-gradient kernel; the weight-
// gradient kernel contracts one against the other over the slots of each sub-module.
// ------------------------------------------------------------------------------------------------
struct TapeLayout {
    // activation tape channels
    int a_pe, a_aux, a_h, a_f, a_g, a_rgb, a_lin, a_sig, a_id, a_total;
    // gradient tape channels
    int g_z, g_final, g_dira, g_rgb, g_sig, g_total;
};

// Sub-matrices of the weights in the layout the data-gradient pass streams them: [n (reduce)][k (out)],
// i.e. the nn.Linear [out,in] storage restricted to the input columns that carry a gradient.
struct BwdLayout {
    int w[MN_MAX_LAYERS];   // [L][L]    layer i >= 1, columns of the hidden part (after the PE block on skip layers)
    int final_w;            // [L][L]
    int dira_f;             // [L/2][L]  dir_a_encoding columns 0..L-1 (the xyz_encoding_final features)
    int dira_e;             // [L/2][app] dir_a_encoding columns of the appearance embedding
    int total;
};

static inline int mn_tape_tm(int L) { return L <= 256 ? 64 : 32; }
// TM-slot tiles one CTA of the fp32 weight-gradient kernel sums before its fp32 atomics (mlp_bwd_weight_kernel)
#define MN_WG_CHUNK_TILES 64

// ---- tensor-core execution plan of a network (csrc/mn_mlp_tc.cu)
constexpr int kMaxGemm = MN_MAX_LAYERS + 2;     // layer engine: every trunk layer, xyz_encoding_final and dir_a_encoding

enum { SRC_H = 0, SRC_XPE = 1, SRC_XAUX = 2 };
enum { EPI_RELU = 0, EPI_RELU_SIGMA = 1, EPI_LINEAR = 2, EPI_RGB = 3,
       // data-gradient chain (training, mn_train_tc.cuh): plain copy, ReLU mask from the activation tape, mask + sigma-head term
       EPI_D_LINEAR = 4, EPI_D_MASK = 5, EPI_D_MASK_SIGMA = 6 };

struct TcGemm {
    int n;           // MMA N = columns of the weight image (layer engine: the output columns padded to 256-column blocks)
    int nseg;
    int src[2];
    int k[2];        // padded K columns per segment (multiple of 16)
    int w_off;       // byte offset of the weight image inside one precision plane of a sub-module
    int bias_off;    // float offset inside the sub-module's fp32 block
    int img;         // data-gradient plan: tape image of the output (ReLU mask read from the activation record, dZ written)
    int epi;
};

struct TcPlan {
    int n_gemm, n_trunk;
    TcGemm g[kMaxGemm];
    int kpe, kaux;         // padded feature-tile widths
    int plane_bytes;       // bytes of all weight images of one sub-module (one precision plane)
    int f32_floats;        // fp32 block: the biases, sigma_w [L], sigma_b (4) [, the layer engine's rgb head]
    int sigma_w_off;       // float offset of sigma_w in the fp32 block
    int sub_bytes;         // total bytes per sub-module: planes (hi[,lo]) + fp32 block
    int x_tile_bytes;      // bytes of one feature tile image (one plane)
    int L;
    int bstride;           // fused engine: floats reserved per GEMM bias in the fp32 block (256; 512 for the 512-wide network)
    int f32_off;           // byte offset of the fp32 block inside one sub-module's pack (after the hi and lo planes)
};

// ---- the network's Linears in forward order (nerf.py:115-160): trunk layers 0 .. layers-1, xyz_encoding_final,
// dir_a_encoding, rgb.  The forward and data-gradient plans, the weight packs and the weight-gradient items of the backward all
// walk this one table.  Linear j's SRC_H segment reads the output of Linear j - 1 (image j - 1 of a tile's activation record).
struct TcSeg {
    int src;             // SRC_XPE / SRC_XAUX (a segment of the feature tile) or SRC_H (the previous Linear's output)
    int k, k_real;       // padded K columns (multiple of 16); columns that exist in the nn.Linear weight
    int in0;             // first input column of the segment in the nn.Linear weight
};
struct TcLinear {
    int n;               // output features
    int cols;            // columns of the output's activation image (n, or lg_cols(n) on the layer engine)
    int nseg;
    TcSeg seg[2];
    int kin;             // in_features
    int w, b;            // PackedLayout float offsets of the weight and the bias (also their offsets in the gradient block)
    int bwd;             // BwdLayout float offset of the [n][L] sub-matrix the data-gradient chain streams; -1: none
    int epi;             // EPI_RELU, EPI_RELU_SIGMA (last trunk layer), EPI_LINEAR (xyz_encoding_final) or EPI_RGB
};
struct TcLinears {
    int n, n_trunk;
    int kpe, kaux;       // padded feature-tile widths
    int hc, gc;          // columns of the H / F images and of the G image (L and L/2 unless padded for the layer engine)
    TcLinear l[MN_MAX_LAYERS + 3];
};

// The layer engine's activation buffers and rgb head, from the forward plan.  GEMM gi writes ping-pong buffer gi % 2 and reads
// the other one; dir_a_encoding writes G to its own buffer: F went to the other ping-pong buffer, so the head still finds
// H_last for sigma.  The buffers have the padded widths of the activation images (TcLinears::hc, gc).  rgb_w ([rgb_dim][rgb_k])
// and rgb_b follow sigma_w (sigma_k floats) and sigma_b in the fp32 block (build_plan).
enum { LB_ACT0 = 0, LB_ACT1 = 1, LB_G = 2 };
struct LgNet {
    int g_gemm;          // the GEMM that writes LB_G (dir_a_encoding), or -1
    int buf_cols[3];     // columns of each activation buffer (0: unused)
    int h_last;          // buffer of the last trunk activations
    int rgb_src;         // buffer the rgb head reads
    int sigma_k, rgb_k;  // columns the fp32 heads read: L and rgb_in rounded up to 8 (the padding weights are zero)
    int rgb_w_off, rgb_b_off;
    int in(int gi) const { return (gi + 1) & 1; }
    int out(int gi) const { return gi == g_gemm ? LB_G : gi & 1; }
};

enum { TC_NONE = 0, TC_FUSED = 1, TC_LAYER = 2 };
struct TcNet {
    int engine;              // TC_NONE (fp32 only), TC_FUSED (tc_mlp_wg_kernel) or TC_LAYER (one GEMM launch per Linear)
    bool train;              // tensor-core training covers the shape (once the weights are packed: tc_packed)
    TcLinears lin;
    TcPlan P;                // engine != TC_NONE: the forward GEMMs and the layout of the forward weight images (tc_packed)
    TcPlan D;                // train: the data-gradient chain and the layout of the transposed weight images (tc_dgrad)
    LgNet lg;                // engine == TC_LAYER: its activation buffers and rgb head
    int64_t act_tile_bytes;  // bytes of one tile's activation record (and of the backward's gradient record)
};

struct mn_model {
    mn_ctx* ctx = nullptr;
    mn_model_desc d{};
    NetDims nd{};
    PackedLayout lay{};
    TapeLayout tape{};
    BwdLayout blay{};
    float* packed = nullptr;          // [n_sub * lay.total] fp32
    float* packed_bwd = nullptr;      // [n_sub * blay.total] fp32, see BwdLayout
    float* centroids_d = nullptr;     // [n_sub, 3]
    int* counters_d = nullptr;        // routing scratch: see mn_route.cu
    int max_multiplicity = 0;         // slot capacity per row for blended routing
    TcNet tc{};                       // tensor-core plan: fixed by nd, lay and blay, so build_layout computes it (tc_net) once
    // tensor-core packed weights (fp16 hi / lo images, mn_mlp_tc.cu): NULL before the first mn_model_set_weights or if TC_NONE
    void* tc_packed = nullptr;
    // transposed fp16 weight images of the tensor-core data-gradient chain (mn_train_tc.cuh); NULL if the shape is not covered
    void* tc_dgrad = nullptr;
    // weights bound by mn_model_bind_weights: per sub-module, the re-layouts of launch 0 (fp32 layouts) and launch 1 (the fp16
    // images that read them), and, once every sub-module is bound, their resident table for mn_model_repack (csrc/mn_api.cu)
    std::vector<std::vector<PackOp>> bound_ops[2];
    std::vector<char> bound;
    std::vector<char> bound_dgrad;      // per sub-module: bound with the transposed images of the backward (tc_dgrad) in its ops
    PackOp* repack_ops = nullptr;       // [n_ops[0] + n_ops[1]]
    long long* repack_first = nullptr;  // per launch: first chunk of each op, then the launch's chunk count [n_ops + 1]
    int repack_n[2] = {0, 0};
    long long repack_chunks[2] = {0, 0};
    std::vector<PackOp> repack_host_ops;        // the table's contents
    std::vector<long long> repack_host_first;
    std::vector<void*> repack_retired;          // earlier tables, which captured graphs may still read (freed with the model)
};

// counters_d layout (ints)
#define CNT_COUNT 0                        // [MN_MAX_SUB]   rows routed to each sub-module
#define CNT_START (MN_MAX_SUB)             // [MN_MAX_SUB+1] tile-aligned slot offsets
#define CNT_CURSOR (2 * MN_MAX_SUB + 1)    // [MN_MAX_SUB]
#define CNT_NSLOTS (3 * MN_MAX_SUB + 1)    // [1] padded slot count (end of last bucket)
#define CNT_NPAIRS (3 * MN_MAX_SUB + 2)    // [1] routed (row, sub) pairs
#define CNT_TICKET (3 * MN_MAX_SUB + 3)    // [1] blocks of the count pass that have finished (the last one scans)
#define CNT_TOTAL (3 * MN_MAX_SUB + 4)

// Arguments common to both MLP kernels.
struct MlpArgs {
    NetDims nd;
    PackedLayout lay;
    const float* packed;      // fp32 packed weights, sub s at packed + s * lay.total
    RowSrc src;
    const int* slot_row;      // slot -> row, -1 = padding; NULL = identity
    const float* slot_w;      // slot -> blend weight; NULL = 1
    const int* counters;      // routing counters (bucket starts, n_slots) or NULL
    int n_sub;
    int fixed_sub;            // used when counters == NULL
    int64_t B;                // rows (identity mode) / slot capacity (routed mode)
    int sigma_only;
    const float* sigma_noise; // [rows] or NULL
    float* out;               // [*, out_cols]
    int out_cols;
    int scatter;              // 1: out index = row, 0: out index = slot
    float* tape;              // activation tape (training forward) or NULL
    TapeLayout tl;
    LiveRows live;            // unrouted calls: rows that hold data (routed calls: the router skips the others)

    // slots that hold rows: the routed slot count, else the live rows
    __device__ __forceinline__ int64_t n_slots() const { return counters ? (int64_t)counters[CNT_NSLOTS] : live.rows(B); }
    // sub-module that owns the 128-slot tile `tile` (routed: the bucket it lies in)
    __device__ __forceinline__ int sub_of_tile(int64_t tile) const {
        int sub = fixed_sub;
        if (counters) {
            sub = 0;
            const int64_t s0 = tile * MN_TILE;
            while (sub + 1 < n_sub && s0 >= counters[CNT_START + sub + 1]) ++sub;
        }
        return sub;
    }
    // row held by `slot`, -1 for padding and for slots at or past n_slots
    __device__ __forceinline__ int64_t row_of_slot(int64_t slot, int64_t n_slots) const {
        int64_t row = -1;
        if (slot < n_slots) row = slot_row ? (int64_t)slot_row[slot] : slot;
        return row;
    }
};

// Arguments of the backward kernels (csrc/mn_backward.cu).
struct BwdArgs {
    NetDims nd;
    PackedLayout lay;
    BwdLayout blay;
    TapeLayout tl;
    const float* packed;       // forward weights (K-major), small heads are read from here
    const float* packed_bwd;   // see BwdLayout
    const int* slot_row;       // slot -> row, -1 = padding; NULL = identity
    const float* slot_w;       // slot -> blend weight; NULL = 1
    const int* counters;       // routing counters SAVED by the forward pass, or NULL
    int n_sub;
    int fixed_sub;
    int64_t B;                 // rows (identity mode) / slot capacity (routed mode)
    const float* grad_out;     // [rows, out_cols]
    int64_t grad_rows;         // rows of grad_out (the model call's B)
    int out_cols;
    const float* act;          // activation tape
    float* grad;               // gradient tape
    float* gw;                 // parameter gradients, [n_sub * lay.total], matrices stored [out][in] (nn.Linear layout)
    // rows of grad_out that hold data, as the recording forward's (the background pass of mn_render_rays_train_bg): unrouted
    // calls run no slot at or past live.rows(B), whose tape was never written; routed calls take their slots from the counters
    LiveRows live;
};

int mn_route_build(mn_ctx* ctx, mn_model* m, const RowSrc& src, int64_t B, LiveRows live, int64_t cap, int* slot_row, float* slot_w,
                   int* row_slots, void* scratch, cudaStream_t st);
size_t mn_route_scratch_bytes(const mn_model* m, int64_t B);   // per-row active-set masks (+ blend weights [K][B])
int mn_route_combine(mn_ctx* ctx, mn_model* m, int64_t B, LiveRows live, const int* row_slots, const float* slot_out, int out_cols,
                     float* out, cudaStream_t st);
// Buckets of an owner call (mn_model_forward_assigned): n rows of `stride` floats whose column id_col holds the sub-module
// (-1 = empty slot) and, if has_noise, column id_col + 1 the density noise, copied to *noise_out (inside `scratch`).
size_t mn_route_assigned_scratch_bytes(int64_t n);
int mn_route_build_assigned(mn_ctx* ctx, mn_model* m, const float* rows, int64_t n, int stride, int id_col, int has_noise, int64_t cap,
                            int* slot_row, void* scratch, const float** noise_out, cudaStream_t st);
// mn_model_forward (inference) over the first live.rows(B) of B rows: the router, the encoders and the MLP tiles see only those,
// the launch sequence is the one for B rows (csrc/mn_api.cu)
// gather (ray-structured rows only): row r is sample gather[r] of `rows` - point gather[r], ray gather[r] / samples_per_ray - and
// its result goes to out_d row r (the queried samples of an occupancy grid, mn_render.cu)
int mn_model_forward_live(mn_ctx* ctx, mn_model* m, const mn_rows* rows, int64_t B, LiveRows live, int use_coarse, int precision,
                          float* out_d, void* workspace_d, size_t workspace_bytes, cudaStream_t st, const int* gather = nullptr);
// The recording forward (mn_model_forward_train(_tc), precision MN_PREC_FP32 / MN_PREC_TC_F16) and its backward (mn_model_backward(_tc))
// over the first live.rows(B) of B rows, with the tape and workspaces of B rows: no slot at or past the live rows is encoded,
// recorded or contracted into a weight gradient, and rows of grad_out past them are never read.  gather: as for
// mn_model_forward_live; sigma_noise_d, the tape and grad_out are indexed by gathered row r, not by sample.
int mn_model_forward_train_live(mn_ctx* ctx, mn_model* m, const mn_rows* rows, int64_t B, LiveRows live, int use_coarse,
                                const float* sigma_noise_d, int precision, float* out_d, void* tape_d, size_t tape_bytes,
                                void* workspace_d, size_t workspace_bytes, cudaStream_t st, const int* gather = nullptr);
int mn_model_backward_live(mn_ctx* ctx, mn_model* m, int64_t B, LiveRows live, int use_coarse, int precision, const float* grad_out_d,
                           const void* tape_d, size_t tape_bytes, float* param_grads_d, void* workspace_d, size_t workspace_bytes,
                           cudaStream_t st);
// ---- the one launch of each stage kernel (csrc/mn_sample.cu).  The public stage entry points validate their arguments and call
// these; the render passes of mn_render_rays(_bg) call them directly, the background pass with its device ray count (`live`: rays
// at or past it are skipped, grids stay sized for N) and the sample orders it needs: flip = reversed stratify output, flip_pts =
// points in reversed sample order (depth_real in sample order), out_flip_d = a second, reversed copy of sort_cat's output.
int mn_stage_stratify(mn_ctx* ctx, const float* z_d, int64_t z_row_stride, const float* rand_d, float perturb, int64_t N, int S, int flip,
                      LiveRows live, float* z_out_d, cudaStream_t st);
int mn_stage_points_outside(mn_ctx* ctx, const float* rays_d, const int64_t* ray_ids_d, const float* depth_d, const float* center3_d,
                            const float* radius3_d, int64_t n, int S, int include_xyz_real, int cluster_2d, int flip_pts, LiveRows live,
                            float* pts_out_d, float* depth_real_out_d, cudaStream_t st);
int mn_stage_sample_pdf(mn_ctx* ctx, const float* z_coarse_d, const float* weights_d, int64_t w_stride, const float* cdf_d, const float* u_d,
                        int64_t u_row_stride, int64_t N, int S, int F, LiveRows live, float* z_out_d, int64_t* inds_out_d,
                        float* cdf_out_d, cudaStream_t st);
int mn_stage_sort_cat(mn_ctx* ctx, const float* a_d, int na, const float* b_d, int nb, int64_t N, int descending, LiveRows live,
                      float* out_d, float* out_flip_d, cudaStream_t st);
int mn_stage_composite(mn_ctx* ctx, const float* raw_d, const float* z_d, const float* depth_real_d, int S, const float* raw2_d,
                       const float* z2_d, const float* depth_real2_d, int S2, const float* last_delta_d, int64_t N, int flip,
                       LiveRows live, float* weights_out_d, float* rgb_out_d, float* depth_out_d, float* depth_var_out_d,
                       float* bg_lambda_out_d, cudaStream_t st);
int mn_stage_sh_to_rgb(mn_ctx* ctx, int deg, const float* coef_d, int64_t coef_stride, const float* dirs_d, int64_t dir_stride,
                       int dir_div, int64_t B, int apply_sigmoid, LiveRows live, float* out_d, cudaStream_t st,
                       const int* gather = nullptr);   // gather: row b's direction is that of sample gather[b] (occupancy grids)
int mn_stage_composite_backward(mn_ctx* ctx, const float* raw_d, const float* z_d, int S, const float* raw2_d, const float* z2_d, int S2,
                                const float* last_delta_d, int64_t N, int flip, LiveRows live, const float* grad_rgb_d,
                                const float* grad_lambda_d, float* grad_raw_d, float* grad_raw2_d, cudaStream_t st);
int mn_stage_sh_to_rgb_backward(mn_ctx* ctx, int deg, const float* coef_d, int64_t coef_stride, const float* dirs_d, int64_t dir_stride,
                                int dir_div, int64_t B, int apply_sigmoid, LiveRows live, const float* grad_out_d, float* grad_coef_d,
                                cudaStream_t st, const int* gather = nullptr);   // gather: as for mn_stage_sh_to_rgb
int mn_mlp_simt_launch(mn_ctx* ctx, const MlpArgs& a, int64_t n_tiles128, cudaStream_t st);
int mn_mlp_bwd_launch(mn_ctx* ctx, const BwdArgs& a, int64_t n_tiles128, cudaStream_t st);
int mn_mlp_tc_launch(mn_ctx* ctx, mn_model* m, const MlpArgs& a, int64_t n_tiles128, int precision, void* ws,
                     size_t ws_bytes, cudaStream_t st);
size_t mn_mlp_tc_workspace(const mn_model* m, int64_t n_tiles128, int precision);
TcNet tc_net(const mn_model& m);
int mn_mlp_tc_pack(mn_ctx* ctx, mn_model* m, int sub, cudaStream_t st);
// host only (test hook): mode 0 inference, 1 recording forward, 2 data-gradient chain (MN_TP_* in mn_b200.h)
int mn_mlp_tp_program(const mn_model& m, int mode, unsigned int* table_out, int cap_entries, int* info8);
// ---- tensor-core training path (csrc/mn_train_tc.cuh): per-tile tape records and the two passes
// An activation record (and the backward pass's gradient record, same layout) holds fp16 images in the layout of the MLP
// kernel's activation buffer, [cols/8][128 slots][8], one every cols * 128 * 2 bytes: H_0 .. H_{layers-1}, then F
// (xyz_encoding_final) at image `layers`, then G (dir_a_encoding, L/2 columns) at image `layers + 1`.  cols = L on the fused
// engine; the layer engine pads L and L/2 to a multiple of 128 columns (zeros), so a 4096-wide, 8-layer record holds about
// 78 KB per sample.
__host__ __device__ __forceinline__ size_t mn_tc_img_off(int img, int cols) { return (size_t)img * cols * MN_TILE * 2; }
// rows of the per-tile fp32 head block [MN_TC_F32_ROWS][128]: sigma pre-activation, rgb (3), image id
enum { MN_TC_F32_SIGMA = 0, MN_TC_F32_RGB = 1, MN_TC_F32_ID = 4, MN_TC_F32_ROWS = 5 };
// rows of the backward pass's per-tile fp32 head-gradient block [mn_tc_g32_rows(rgb_dim)][128]: d sigma pre-activation, d rgb
// pre-activation (rgb_dim rows: 3 colour channels before the sigmoid, or the raw SH coefficients).
// Bounds of rgb_dim (register and shared-memory arrays of the head kernels are sized by them): MN_TC_RGB_MAX for the fused
// engine (its rgb head is an N = 32 GEMM), MN_TC_LG_RGB_MAX for the layer-GEMM engine's CUDA-core head (SH degree 4: 75
// coefficients).  The layer engine's head kernels come in both sizes; mn_tc_lg_rgb_bound picks the one a network runs.
enum { MN_TC_G32_SIGMA = 0, MN_TC_G32_RGB = 1, MN_TC_RGB_MAX = 32, MN_TC_LG_RGB_MAX = 80 };
__host__ __device__ __forceinline__ int mn_tc_g32_rows(int rgb_dim) { return 1 + rgb_dim; }
__host__ __device__ __forceinline__ int mn_tc_lg_rgb_bound(int rgb_dim) { return rgb_dim <= MN_TC_RGB_MAX ? MN_TC_RGB_MAX : MN_TC_LG_RGB_MAX; }
struct TrainTcTape {
    unsigned char* xreg;      // encoder feature tiles        [n_tiles][x_tile_bytes]
    unsigned char* act;       // activation records           [n_tiles][act_tile_bytes]
    float* f32;               // fp32 head blocks             [n_tiles][MN_TC_F32_ROWS][128]
};
// the shapes whose recording calls run on the tensor cores (tc_net in mn_mlp_tc.cu; mn_model_train_tc_supported)
#define MN_TC_TRAIN_COVERAGE                                                                                                     \
    "tensor-core training covers layer_dim 256..4096 with 2..16 layers and a direction / appearance head, "                       \
    "rgb_dim 3 or a raw SH head (rgb_dim <= 80: sh_deg <= 4), no affine appearance; use train precision 'fp32'"
// the recording forward into `tape`: of a training call (train, the caller has checked m->tc.train && m->tc_packed) or of the
// test hook, which runs every network with a tensor-core forward
int mn_mlp_tc_launch_record(mn_ctx* ctx, mn_model* m, const MlpArgs& a, int64_t n_tiles128, const TrainTcTape& tape, bool train,
                            cudaStream_t st);
size_t mn_train_tc_backward_workspace(const mn_model* m, int64_t n_tiles128);
// host only (test hook mn_debug_tc_train_layout): the entries MN_TCL_ENGINE .. that the engine decides
int mn_train_tc_layout(const mn_model* m, int64_t n_tiles128, int64_t* out, int cap);
int mn_train_tc_backward(mn_ctx* ctx, mn_model* m, const BwdArgs& a, int64_t n_tiles128, const TrainTcTape& tape, void* ws, size_t ws_bytes,
                         cudaStream_t st);
