// mn_render_rays / mn_render_rays_bg: the inference path of render_rays (rendering.py:15-248, eval mode) as ONE C call.  Each
// network is rendered by one two-pass routine, as the reference's _get_results (rendering.py:176-248): coarse query ->
// composite -> inverse-CDF resampling -> fine query -> merge + volume rendering.  The foreground pass runs it on all rays; with
// a background (NeRF++) network (rendering.py:34-62, 143-173) a sphere split comes first, the background pass runs it flipped
// on the inverted-sphere points of the compacted background rays, and a lambda blend comes last.  The call only sequences the
// stage kernels of this library on the caller's stream, from a caller-provided workspace: no allocation, no host sync, ~20
// (foreground) / ~40 (with background) launches issued back to back without returning to the host language in between (the
// Python mirror spends 1.6-2.0 ms of interpreter time on the foreground alone).
//
// The background rays are compacted on the device (stable: ascending ray order) and their count stays there: every kernel of
// the background pass - stages, router, encoders, MLP tiles - skips rays / rows past it, while grids are sized for all N rays.
// So the launch sequence is static (CUDA-graph capturable) and the background work follows the live count.  A camera outside
// the ellipsoid sets the context's status word (MN_ERR_SPHERE at the next mn_check_status), as mn_intersect_sphere does.
#include "mn_model.cuh"

namespace {

__global__ void fill_kernel(float* p, int64_t n, float v) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}

// torch.maximum / torch.minimum: NaN-propagating
__device__ __forceinline__ float max_t(float a, float b) { return a != a ? a : (b != b ? b : (a < b ? b : a)); }
__device__ __forceinline__ float min_t(float a, float b) { return a != a ? a : (b != b ? b : (b < a ? b : a)); }

// Threads per block of the split and occupancy-test kernels and of the compaction that follows each: a count per block, then a
// stable scan over the counts of the blocks before (compact_block_scan).
constexpr int kCompactBlock = 1024;

// The stable block scan of a compaction (torch.arange(n)[mask] order) in a kCompactBlock-thread block: keep = this thread's element
// stays, blk[b] = elements kept in block b.  Returns the element's compacted position, -1 if it is not kept; the last block writes
// the number kept to *count (and to *count_out if given).
__device__ __forceinline__ int compact_block_scan(const int* __restrict__ blk, bool keep, int* __restrict__ count,
                                                  int* __restrict__ count_out) {
    __shared__ int wsum[32], wbase[32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int part = 0;                                           // elements kept in the blocks before this one
    for (unsigned b = threadIdx.x; b < blockIdx.x; b += kCompactBlock) part += blk[b];
    for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
    const unsigned bal = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) { wsum[warp] = part; wbase[warp] = __popc(bal); }
    __syncthreads();
    if (threadIdx.x == 0) {
        int run = 0;
        for (int w = 0; w < kCompactBlock / 32; ++w) run += wsum[w];
        for (int w = 0; w < kCompactBlock / 32; ++w) { const int c = wbase[w]; wbase[w] = run; run += c; }
        if (blockIdx.x == gridDim.x - 1) {
            *count = run;
            if (count_out) *count_out = run;
        }
    }
    __syncthreads();
    return keep ? wbase[warp] + __popc(bal & ((1u << lane) - 1)) : -1;
}

// Background split, per ray (render.py `_render`, rendering.py:34-47): fg_far = max(sphere exit, near); the ray reaches the
// background iff far > fg_far; its last delta (fg_far, else 1e10) and the foreground far override min(far, fg_far).  flag[i] = 1
// for a background ray (turned into its compacted position by bg_compact_kernel); blk[b] = background rays of block b.
__global__ void __launch_bounds__(kCompactBlock) bg_split_kernel(const float* __restrict__ rays, const float* __restrict__ center,
                                                                 const float* __restrict__ radius, int64_t N, float* __restrict__ far_ov,
                                                                 float* __restrict__ last_delta, int* __restrict__ flag,
                                                                 int* __restrict__ blk, unsigned int* status) {
    const int64_t i = (int64_t)blockIdx.x * kCompactBlock + threadIdx.x;
    bool with_bg = false;
    if (i < N) {
        const float* r = rays + i * 8;
        bool outside;
        const float fg_far = max_t(mn_sphere_far(r, center, radius, &outside), r[6]);
        const float far = r[7];
        if (outside) {
            // camera not bounded by the ellipsoid: the status word carries the error (the call's results are undefined); the
            // sphere exit is NaN here, so the ray is rendered as foreground-only up to its own far bound, keeping every depth
            // the later passes sort and merge finite
            atomicOr(status, MN_STATUS_SPHERE);
            last_delta[i] = 1e10f;
            far_ov[i] = far;
        } else {
            with_bg = far > fg_far;
            last_delta[i] = with_bg ? fg_far : 1e10f;
            far_ov[i] = min_t(far, fg_far);
        }
        flag[i] = with_bg ? 1 : 0;
    }
    const int n = __syncthreads_count(with_bg);
    if (threadIdx.x == 0) blk[blockIdx.x] = n;
}

// Stable compaction of the background rays (torch.arange(N)[mask]): ids, directions and image indices of the compacted rays,
// pos[i] = compacted position of ray i or -1, *count = number of background rays (written by the last block).
__global__ void __launch_bounds__(kCompactBlock) bg_compact_kernel(const float* __restrict__ rays, const float* __restrict__ idx,
                                                                   int64_t N, const int* __restrict__ blk, int* __restrict__ pos,
                                                                   int64_t* __restrict__ ids, float* __restrict__ dirs,
                                                                   float* __restrict__ cidx, int* __restrict__ count) {
    const int64_t i = (int64_t)blockIdx.x * kCompactBlock + threadIdx.x;
    const int p = compact_block_scan(blk, i < N && pos[i] != 0, count, nullptr);
    if (i >= N) return;
    if (p >= 0) {
        ids[p] = i;
        for (int j = 0; j < 3; ++j) dirs[p * 3 + j] = rays[i * 8 + 3 + j];
        if (cidx) cidx[p] = idx[i];
    }
    pos[i] = p;
}

// Lambda blend of one result (render.py `_render`, rendering.py:60-62): add = bg_val * bg_lambda for a background ray, 0 for the
// others; val + add with both operations separately rounded, as torch's two ops.  Optionally fg_* = val and bg_* = add.
__global__ void bg_blend_kernel(float* __restrict__ val, const float* __restrict__ bg_val, const float* __restrict__ lam,
                                const int* __restrict__ pos, int64_t N, int C, float* __restrict__ fg_out, float* __restrict__ bg_out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N * C) return;
    const int64_t ray = i / C;
    const int p = pos[ray];
    const float v = val[i];
    const float add = p >= 0 ? __fmul_rn(bg_val[(int64_t)p * C + (i - ray * C)], lam[ray]) : 0.0f;
    if (fg_out) fg_out[i] = v;
    if (bg_out) bg_out[i] = add;
    val[i] = __fadd_rn(v, add);
}

// ---- occupancy grid (mn_render_rays_occ / mn_render_rays_bg_occ): the foreground samples in cells the grid marks empty are not
// queried, their raw row is (0, 0, 0, 0).  The queried samples are compacted on the device like the background rays (a block
// count, then a stable block scan over the counts of the blocks before), the model runs on them through a row gather with its
// row count read from the device, and a scatter writes every raw row.
struct OccGrid {
    const uint32_t* bits;   // reso^3 bits, cell (i * reso + j) * reso + k at bit c & 31 of word c >> 5
    int reso;
    float off[3], scl[3];
};

// Whether the sample at p[0..2] is queried.  u_a = p_a * scale_a + offset_a is two separately rounded fp32 operations (no FMA,
// __fmul_rn / __fadd_rn), the cell index floorf(u_a * reso).  A point outside [0, 1)^3 - NaN included, which fails both
// comparisons - is always queried.  u_a < 1 keeps u_a * reso below reso in fp32 (round-to-nearest is monotone and
// (1 - 2^-24) * reso rounds below reso), so the min() never binds; it only keeps the read inside the grid.
__device__ __forceinline__ bool occ_queried(const OccGrid& g, const float* __restrict__ p) {
    int64_t cell = 0;
    for (int a = 0; a < 3; ++a) {
        const float u = __fadd_rn(__fmul_rn(p[a], g.scl[a]), g.off[a]);
        if (!(u >= 0.0f && u < 1.0f)) return true;
        const int i = min((int)floorf(__fmul_rn(u, (float)g.reso)), g.reso - 1);
        cell = cell * g.reso + i;
    }
    return (g.bits[cell >> 5] >> (cell & 31)) & 1u;
}

// flag[s] = 1 iff sample s of the [n, 3] points is queried; blk[b] = queried samples of block b.
__global__ void __launch_bounds__(kCompactBlock) occ_test_kernel(const float* __restrict__ xyz, int64_t n, OccGrid g,
                                                                 int* __restrict__ flag, int* __restrict__ blk) {
    const int64_t s = (int64_t)blockIdx.x * kCompactBlock + threadIdx.x;
    bool q = false;
    if (s < n) {
        q = occ_queried(g, xyz + s * 3);
        flag[s] = q ? 1 : 0;
    }
    const int c = __syncthreads_count(q);
    if (threadIdx.x == 0) blk[blockIdx.x] = c;
}

// Stable compaction of the queried samples: idx[0 .. count) = their flat indices in ascending order, pos[s] = the compacted row
// of sample s or -1, *count (and *count_out if given) = the queried samples (written by the last block).  noise_cmp (training,
// when given): noise_cmp[p] = noise[idx[p]], the density noise of each queried sample at its compacted row, where the MLP reads it.
__global__ void __launch_bounds__(kCompactBlock) occ_compact_kernel(int64_t n, const int* __restrict__ blk, int* __restrict__ pos,
                                                                    int* __restrict__ idx, int* __restrict__ count,
                                                                    int* __restrict__ count_out, const float* __restrict__ noise,
                                                                    float* __restrict__ noise_cmp) {
    const int64_t s = (int64_t)blockIdx.x * kCompactBlock + threadIdx.x;
    const int p = compact_block_scan(blk, s < n && pos[s] != 0, count, count_out);
    if (s >= n) return;
    if (p >= 0) {
        idx[p] = (int)s;
        if (noise_cmp) noise_cmp[p] = noise[s];
    }
    pos[s] = p;
}

// raw[s] = the compacted result row pos[s], or (0, 0, 0, 0) for a sample that was not queried.
__global__ void occ_scatter_kernel(const float4* __restrict__ cmp, const int* __restrict__ pos, int64_t n, float4* __restrict__ raw) {
    const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    const int p = pos[s];
    raw[s] = p >= 0 ? cmp[p] : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
}

// bits[w] = the cells 32 w .. 32 w + 31 with sigma >= thresh (mn_occupancy_pack): lane l of a warp holds cell 32 w + l, so the
// ballot is the word; cells past n are empty.
__global__ void occ_pack_kernel(const float* __restrict__ sigma, int64_t n, float thresh, uint32_t* __restrict__ bits) {
    const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned word = __ballot_sync(0xffffffffu, c < n && sigma[c] >= thresh);
    if ((threadIdx.x & 31) == 0 && c < n) bits[c >> 5] = word;
}

// Workspace offsets: each buffer aligned on its own.
struct Carve {
    size_t off = 0;
    size_t operator()(size_t bytes) { const size_t o = off; off += mn_align(bytes); return o; }
};

constexpr size_t kNone = ~(size_t)0;   // offset of a buffer the pass does not use

// The buffers of one two-pass render over N rays: S coarse samples, F fine draws, Sq samples of the fine query (F, or S + F
// under cascade).  z_c / z_q hold the coarse / fine-query depths in sample order, from which the fine draws are resampled and
// the points made.  z_c_comp / z_q_comp hold them as the composite reads them: the same buffers, or with flip (the background
// pass) reversed copies of the coarse depths and, under cascade, of the fine-query depths.  With flip, dreal_c / dreal_f are
// the real depths of the points outside the sphere.
struct PassBufs {
    int S, F, Sq, flip;
    size_t z_c, z_c_comp, xyz_c, dreal_c, mlp_c, raw_c, w_c, z_f, z_q, z_q_comp, xyz_f, dreal_f, mlp_f, raw_f;
    size_t model_ws_bytes;     // model workspace of the larger of the pass's two queries
};

// pt_cols: columns of the pass's points (3 for the foreground, up to 7 for the background).
PassBufs carve_pass(Carve& take, const mn_model* net, int64_t N, int S, int F, int use_cascade, bool sh, int pt_cols, bool flip,
                    int precision) {
    PassBufs b{};
    b.S = S; b.F = F; b.flip = flip;
    b.Sq = F > 0 ? (use_cascade ? S + F : F) : 0;
    const int Sc = S > 0 ? S : 1, Sq = b.Sq > 0 ? b.Sq : 1, out_cols = net->nd.rgb_dim + 1;
    b.z_c = take((size_t)N * Sc * 4);
    b.z_c_comp = flip ? take((size_t)N * Sc * 4) : b.z_c;
    b.xyz_c = take((size_t)N * Sc * pt_cols * 4);
    b.dreal_c = flip ? take((size_t)N * Sc * 4) : kNone;
    b.mlp_c = sh ? take((size_t)N * Sc * out_cols * 4) : kNone;      // raw SH coefficients before the head
    b.raw_c = take((size_t)N * Sc * 16);
    b.w_c = take((size_t)N * Sc * 4);
    b.z_f = take((size_t)N * (F > 0 ? F : 1) * 4);
    b.z_q = use_cascade && F > 0 ? take((size_t)N * Sq * 4) : b.z_f;
    b.z_q_comp = flip && use_cascade && F > 0 ? take((size_t)N * Sq * 4) : b.z_q;
    b.xyz_f = take((size_t)N * Sq * pt_cols * 4);
    b.dreal_f = flip ? take((size_t)N * Sq * 4) : kNone;
    b.mlp_f = sh ? take((size_t)N * Sq * out_cols * 4) : kNone;
    b.raw_f = take((size_t)N * Sq * 16);
    const size_t a = mn_model_workspace_bytes(net, N * Sc, precision);
    const size_t c = b.Sq > 0 ? mn_model_workspace_bytes(net, N * b.Sq, precision) : 0;
    b.model_ws_bytes = a > c ? a : c;
    return b;
}

struct RenderPlan {
    PassBufs fg, bg;
    size_t last_delta, model_ws, model_ws_bytes, total;
    // occupancy grid (foreground queries, sized for the larger of the two): flags / compacted rows, sample indices, block counts,
    // the queried-row count of each pass, compacted results [rows, 4]
    size_t occ_pos, occ_idx, occ_blk, occ_count, occ_out;
    // background split and blend; every per-ray buffer holds N rays (the compacted background rays first)
    size_t far_ov, pos, blk, count, ids, dirs, idx, ld_b, rgb_b, depth_b, rgb_cb, lam, lam_c;
};

RenderPlan make_plan(const mn_model* m, const mn_model* bg, int64_t N, int Sc, int Sf, int use_cascade, int sh, int precision,
                     bool occ = false) {
    RenderPlan p{};
    Carve take;
    p.fg = carve_pass(take, m, N, Sc, Sf, use_cascade, sh, 3, false, precision);
    p.last_delta = take((size_t)N * 4);
    if (occ) {
        const int64_t rows = N * (p.fg.Sq > Sc ? p.fg.Sq : Sc);
        p.occ_pos = take((size_t)rows * 4);
        p.occ_idx = take((size_t)rows * 4);
        p.occ_blk = take((size_t)mn_cdiv(rows, kCompactBlock) * 4);
        p.occ_count = take(2 * 4);
        p.occ_out = take((size_t)rows * 16);
    }
    p.model_ws_bytes = p.fg.model_ws_bytes;
    if (bg) {
        p.far_ov = take((size_t)N * 4);
        p.pos = take((size_t)N * 4);
        p.blk = take((size_t)mn_cdiv(N, kCompactBlock) * 4);
        p.count = take(4);
        p.ids = take((size_t)N * 8);
        p.dirs = take((size_t)N * 12);
        p.idx = take((size_t)N * 4);
        // half the samples (rendering.py:47-48); 7 point columns with the real-xyz prefix, else 4
        p.bg = carve_pass(take, bg, N, Sc / 2, Sf / 2, use_cascade, sh, 7, true, precision);
        p.ld_b = take((size_t)N * 4);
        p.rgb_b = take((size_t)N * 12);
        p.depth_b = take((size_t)N * 4);
        p.rgb_cb = take((size_t)N * 12);
        p.lam = take((size_t)N * 4);
        p.lam_c = take((size_t)N * 4);
        if (p.bg.model_ws_bytes > p.model_ws_bytes) p.model_ws_bytes = p.bg.model_ws_bytes;
    }
    p.model_ws = take(p.model_ws_bytes);
    p.total = take.off + 256;
    return p;
}

// The checks a network of the render passes; name: the entry point, for the message.
int check_net(mn_ctx* ctx, const mn_model* m, int use_cascade, int fine_samples, int sh_deg, const float* image_indices_d,
              const char* name) {
    const mn_model_desc& d = m->d;
    const std::string n(name);
    if (sh_deg >= 0 && (d.pos_dir_dim != 0 || d.rgb_dim != 3 * (sh_deg + 1) * (sh_deg + 1) || sh_deg > 4))
        return mn_fail(ctx, MN_ERR_INVALID, n + ": sh_deg does not match the model's rgb_dim (model_utils.py:58)");
    if (sh_deg < 0 && d.rgb_dim != 3) return mn_fail(ctx, MN_ERR_INVALID, n + ": rgb_dim > 3 needs sh_deg");
    if ((d.kind == 1) != (use_cascade != 0)) return mn_fail(ctx, MN_ERR_INVALID, n + ": use_cascade must match the model kind");
    if (!use_cascade && fine_samples == 0)
        return mn_fail(ctx, MN_ERR_INVALID, n + ": a coarse-only render composites colour only under use_cascade (rendering.py:199)");
    if (d.appearance_dim > 0 && !image_indices_d) return mn_fail(ctx, MN_ERR_INVALID, n + ": image indices are required");
    return MN_OK;
}

// The background split and the compaction of the background rays (render.py `_render`), then the background pass's last deltas
// (1e10: that pass has no bg_lambda).  far_ov, last_delta: the foreground's far override and last deltas; pos, blk, count, ids,
// dirs, idx (null: no image indices): the split and the compacted rays, as bg_split_kernel / bg_compact_kernel; ld_b: the
// background's last deltas.
int split_bg(mn_ctx* ctx, const float* rays_d, const float* image_indices_d, int64_t N, const float* center_d, const float* radius_d,
             float* far_ov, float* last_delta, int* pos, int* blk, int* count, int64_t* ids, float* dirs, float* idx, float* ld_b,
             cudaStream_t st) {
    const unsigned nblk = (unsigned)mn_cdiv(N, kCompactBlock);
    bg_split_kernel<<<nblk, kCompactBlock, 0, st>>>(rays_d, center_d, radius_d, N, far_ov, last_delta, pos, blk, ctx->status_d);
    MN_LAUNCH_CHECK(ctx);
    bg_compact_kernel<<<nblk, kCompactBlock, 0, st>>>(rays_d, image_indices_d, N, blk, pos, ids, dirs, idx, count);
    MN_LAUNCH_CHECK(ctx);
    fill_kernel<<<(unsigned)mn_cdiv(N, 256), 256, 0, st>>>(ld_b, N, 1e10f);
    MN_LAUNCH_CHECK(ctx);
    return MN_OK;
}

// The lambda blend (render.py `_render`) of o's rgb, its depth when wanted and, given lam_c, its rgb_coarse with the background
// pass's results in bo, by bg_lambda of the final type (lam) and of the cascade's coarse type (lam_c); o's fg_* / bg_* (null:
// not wanted) receive the two terms.
int blend_bg(mn_ctx* ctx, const mn_render_outputs& o, const mn_render_outputs& bo, const float* lam, const float* lam_c,
             const int* pos, int64_t N, cudaStream_t st) {
    auto blend = [&](float* val, const float* bval, const float* l, int C, float* fg_out, float* bg_out) -> int {
        bg_blend_kernel<<<(unsigned)mn_cdiv(N * C, 256), 256, 0, st>>>(val, bval, l, pos, N, C, fg_out, bg_out);
        MN_LAUNCH_CHECK(ctx);
        return MN_OK;
    };
    int rc;
    if ((rc = blend(o.rgb, bo.rgb, lam, 3, o.fg_rgb, o.bg_rgb))) return rc;
    if (o.depth && (rc = blend(o.depth, bo.depth, lam, 1, o.fg_depth, o.bg_depth))) return rc;
    if (lam_c && o.rgb_coarse) return blend(o.rgb_coarse, bo.rgb_coarse, lam_c, 3, o.fg_rgb_coarse, o.bg_rgb_coarse);
    return MN_OK;
}

int render_impl(mn_ctx* ctx, mn_model* m, mn_model* bg, const float* rays_d, const float* image_indices_d, int64_t N,
                const float* center_d, const float* radius_d, int include_xyz_real, int cluster_2d, const float* z_steps_d,
                const float* z_steps_bg_d, int coarse_samples, const float* u_fine_d, const float* u_fine_bg_d, int fine_samples,
                int use_cascade, int sh_deg, int precision, const mn_render_outputs& o, void* workspace_d, size_t workspace_bytes,
                void* stream, const char* name, const mn_occupancy* occ = nullptr, int* counts_out_d = nullptr) {
    const std::string nm(name);
    if (!ctx || !m || !rays_d || !z_steps_d || !o.rgb || N < 0 || coarse_samples < 1 || fine_samples < 0) return MN_ERR_INVALID;
    if (fine_samples > 0 && !u_fine_d) return mn_fail(ctx, MN_ERR_INVALID, nm + ": u_fine_d is required when fine_samples > 0");
    if (fine_samples > 0 && coarse_samples < 3) return mn_fail(ctx, MN_ERR_INVALID, nm + ": resampling needs >= 3 coarse samples");
    int rc;
    if ((rc = check_net(ctx, m, use_cascade, fine_samples, sh_deg, image_indices_d, name))) return rc;
    if (bg) {
        if ((rc = check_net(ctx, bg, use_cascade, fine_samples, sh_deg, image_indices_d, name))) return rc;
        if (!z_steps_bg_d || coarse_samples < 2) return mn_fail(ctx, MN_ERR_INVALID, nm + ": the background pass needs z_steps_bg and >= 2 coarse samples");
        if (fine_samples > 0 && (!u_fine_bg_d || fine_samples < 2 || coarse_samples / 2 < 3))
            return mn_fail(ctx, MN_ERR_INVALID, nm + ": background resampling needs u_fine_bg, >= 2 fine and >= 6 coarse samples");
        if (radius_d && !center_d) return mn_fail(ctx, MN_ERR_INVALID, nm + ": sphere radius without a center");
    }
    if (occ) {
        if (!occ->bits || occ->reso < 1 || occ->reso > MN_OCC_MAX_RESO)
            return mn_fail(ctx, MN_ERR_INVALID, nm + ": the occupancy grid needs bits and a reso of 1.." + std::to_string(MN_OCC_MAX_RESO));
        const int Sq = fine_samples > 0 ? (use_cascade ? coarse_samples + fine_samples : fine_samples) : 0;
        if (N * (int64_t)(Sq > coarse_samples ? Sq : coarse_samples) > INT32_MAX)
            return mn_fail(ctx, MN_ERR_INVALID, nm + ": an occupancy-grid render indexes at most 2^31 - 1 samples per pass");
    }
    if (N == 0) return MN_OK;
    const bool sh = sh_deg >= 0;
    const RenderPlan p = make_plan(m, bg, N, coarse_samples, fine_samples, use_cascade, sh, precision, occ != nullptr);
    if (!workspace_d || workspace_bytes < p.total) return mn_fail(ctx, MN_ERR_WORKSPACE, nm + ": workspace too small");
    char* W = (char*)workspace_d;
    auto F = [&](size_t off) { return off == kNone ? nullptr : reinterpret_cast<float*>(W + off); };
    auto I = [&](size_t off) { return reinterpret_cast<int*>(W + off); };
    cudaStream_t st = (cudaStream_t)stream;
    const bool fine = fine_samples > 0;

    // one model query on [N, S, cols] points -> raw [N, S, 4]   (rendering.py:275-334).  dirs / idx: per ray.
    auto query = [&](mn_model* net, const float* xyz, int cols, int S, int coarse, float* mlp_out, float* raw_out, const float* dirs,
                     int64_t dstride, const float* idx, const int* live) -> int {
        mn_rows rows{};
        rows.mode = 1;
        rows.x_d = xyz;
        rows.cols = cols;
        rows.dirs_d = net->d.pos_dir_dim > 0 ? dirs : nullptr;
        rows.dir_stride = dstride;
        rows.idx_d = net->d.appearance_dim > 0 ? idx : nullptr;
        rows.samples_per_ray = S;
        float* out = sh ? mlp_out : raw_out;
        const LiveRows lr{live, S};
        int r = mn_model_forward_live(ctx, net, &rows, N * S, lr, coarse, precision, out, W + p.model_ws, p.model_ws_bytes, st);
        if (r) return r;
        if (sh) return mn_stage_sh_to_rgb(ctx, sh_deg, mlp_out, net->nd.rgb_dim + 1, dirs, dstride, S, N * S, 1, lr, raw_out, st);
        return MN_OK;
    };

    // The same query of the foreground points through the occupancy grid: test and compaction of the N * S samples, the model
    // (and the SH head) on the queried rows, whose count stays on the device, then every raw row from them or zero.  pass: 0
    // coarse, 1 fine (the slot of the queried-row count).
    OccGrid G{};
    if (occ) {
        G.bits = occ->bits;
        G.reso = occ->reso;
        for (int a = 0; a < 3; ++a) { G.off[a] = occ->offset[a]; G.scl[a] = occ->scale[a]; }
    }
    auto query_occ = [&](mn_model* net, const float* xyz, int S, int coarse, float* mlp_out, float* raw_out, const float* dirs,
                         int64_t dstride, const float* idx, int pass) -> int {
        const int64_t n = N * S;
        const unsigned nblk = (unsigned)mn_cdiv(n, kCompactBlock);
        int* cnt = I(p.occ_count) + pass;
        const int* gather = I(p.occ_idx);
        occ_test_kernel<<<nblk, kCompactBlock, 0, st>>>(xyz, n, G, I(p.occ_pos), I(p.occ_blk));
        MN_LAUNCH_CHECK(ctx);
        occ_compact_kernel<<<nblk, kCompactBlock, 0, st>>>(n, I(p.occ_blk), I(p.occ_pos), I(p.occ_idx), cnt,
                                                           counts_out_d ? counts_out_d + pass : nullptr, nullptr, nullptr);
        MN_LAUNCH_CHECK(ctx);
        mn_rows rows{};
        rows.mode = 1;
        rows.x_d = xyz;
        rows.cols = 3;
        rows.dirs_d = net->d.pos_dir_dim > 0 ? dirs : nullptr;
        rows.dir_stride = dstride;
        rows.idx_d = net->d.appearance_dim > 0 ? idx : nullptr;
        rows.samples_per_ray = S;
        const LiveRows lr{cnt, 1};
        float* cmp = F(p.occ_out);
        int r = mn_model_forward_live(ctx, net, &rows, n, lr, coarse, precision, sh ? mlp_out : cmp, W + p.model_ws, p.model_ws_bytes,
                                      st, gather);
        if (r) return r;
        if (sh && (r = mn_stage_sh_to_rgb(ctx, sh_deg, mlp_out, net->nd.rgb_dim + 1, dirs, dstride, S, n, 1, lr, cmp, st, gather)))
            return r;
        occ_scatter_kernel<<<(unsigned)mn_cdiv(n, 256), 256, 0, st>>>(reinterpret_cast<const float4*>(cmp), I(p.occ_pos), n,
                                                                      reinterpret_cast<float4*>(raw_out));
        MN_LAUNCH_CHECK(ctx);
        return MN_OK;
    };
    // a query of pass `pass`: through the grid in the foreground pass (masked) when there is one
    auto query_pass = [&](bool masked, mn_model* net, const float* xyz, int cols, int S, int coarse, float* mlp_out, float* raw_out,
                          const float* dirs, int64_t dstride, const float* idx, const int* live, int pass) -> int {
        if (masked) return query_occ(net, xyz, S, coarse, mlp_out, raw_out, dirs, dstride, idx, pass);
        return query(net, xyz, cols, S, coarse, mlp_out, raw_out, dirs, dstride, idx, live);
    };

    // The two-pass render of one network (rendering.py:176-248, render.py `_two_pass`) from the coarse depths and points the
    // caller wrote into b.z_c, b.z_c_comp, b.xyz_c and b.dreal_c.  live: the device count of the rays that hold data (background
    // pass), or null for all N.  cols: point columns.  fine_points(z, S, flip_pts, xyz, dreal) makes the fine points from the
    // fine-query depths (rendering.py `xyz_fine_fn`).  r: rgb, depth, depth_var and bg_lambda of the final type, rgb_coarse and
    // bg_lambda_coarse of the cascade's coarse type (null: not wanted).
    auto two_pass = [&](mn_model* net, const PassBufs& b, const int* live, int cols, const float* last_delta, const float* u_fine,
                        const float* dirs, int64_t dstride, const float* idx, const mn_render_outputs& r, auto&& fine_points) -> int {
        const LiveRows lr{live, 1};
        const bool masked = occ && !b.flip;   // the grid applies to the foreground pass only
        // depth scratch when only the variance is wanted: the coarse weights are dead by the time it is written
        float* depth = r.depth ? r.depth : (r.depth_var ? F(b.w_c) : nullptr);
        int e;
        if ((e = query_pass(masked, net, F(b.xyz_c), cols, b.S, 1, F(b.mlp_c), F(b.raw_c), dirs, dstride, idx, live, 0))) return e;
        if ((e = mn_stage_composite(ctx, F(b.raw_c), F(b.z_c_comp), F(b.dreal_c), b.S, nullptr, nullptr, nullptr, 0, last_delta, N,
                                    b.flip, lr, fine ? F(b.w_c) : nullptr, use_cascade ? (fine ? r.rgb_coarse : r.rgb) : nullptr,
                                    fine ? nullptr : depth, fine ? nullptr : r.depth_var,
                                    use_cascade ? (fine ? r.bg_lambda_coarse : r.bg_lambda) : nullptr, st)))
            return e;
        if (!fine) return MN_OK;
        // resampling from the bins of the depths in sample order, with the weights as composited (quirk Q7)
        if ((e = mn_stage_sample_pdf(ctx, F(b.z_c), F(b.w_c), b.S, nullptr, u_fine, 0, N, b.S, b.F, lr, F(b.z_f), nullptr, nullptr, st)))
            return e;
        if (use_cascade)
            if ((e = mn_stage_sort_cat(ctx, F(b.z_c), b.S, F(b.z_f), b.F, N, 0, lr, F(b.z_q), b.flip ? F(b.z_q_comp) : nullptr, st))) return e;
        if ((e = fine_points(F(b.z_q), b.Sq, b.flip && use_cascade, F(b.xyz_f), F(b.dreal_f)))) return e;
        if ((e = query_pass(masked, net, F(b.xyz_f), cols, b.Sq, 0, F(b.mlp_f), F(b.raw_f), dirs, dstride, idx, live, 1))) return e;
        if (use_cascade)
            return mn_stage_composite(ctx, F(b.raw_f), F(b.z_q_comp), F(b.dreal_f), b.Sq, nullptr, nullptr, nullptr, 0, last_delta, N,
                                      b.flip, lr, nullptr, r.rgb, depth, r.depth_var, r.bg_lambda, st);
        return mn_stage_composite(ctx, F(b.raw_f), F(b.z_q_comp), F(b.dreal_f), b.Sq, F(b.raw_c), F(b.z_c_comp), F(b.dreal_c), b.S,
                                  last_delta, N, b.flip, lr, nullptr, r.rgb, depth, r.depth_var, r.bg_lambda, st);
    };

    mn_render_outputs bo{};     // the background pass's results
    if (!bg) {
        fill_kernel<<<(unsigned)mn_cdiv(N, 256), 256, 0, st>>>(F(p.last_delta), N, 1e10f);   // no background: rendering.py:33
        MN_LAUNCH_CHECK(ctx);
    } else {
        // ---- split and compaction (render.py:292-299)
        float* bidx = image_indices_d ? F(p.idx) : nullptr;
        if ((rc = split_bg(ctx, rays_d, image_indices_d, N, center_d, radius_d, F(p.far_ov), F(p.last_delta), I(p.pos), I(p.blk),
                           I(p.count), reinterpret_cast<int64_t*>(W + p.ids), F(p.dirs), bidx, F(p.ld_b), st)))
            return rc;

        // ---- background pass over the compacted rays (render.py:300-312): coarse depths from z_steps_bg, in sample order and
        // reversed, and the points outside the sphere in reversed order
        const int* cnt = I(p.count);
        const LiveRows lr{cnt, 1};
        const int64_t* ids = reinterpret_cast<const int64_t*>(W + p.ids);
        const PassBufs& b = p.bg;
        auto outside = [&](const float* z, int S, int flip_pts, float* xyz, float* dreal) {
            return mn_stage_points_outside(ctx, rays_d, ids, z, center_d, radius_d, N, S, include_xyz_real, cluster_2d, flip_pts, lr,
                                           xyz, dreal, st);
        };
        if ((rc = mn_stage_stratify(ctx, z_steps_bg_d, 0, nullptr, 0.0f, N, b.S, 0, lr, F(b.z_c), st))) return rc;
        if ((rc = mn_stage_stratify(ctx, z_steps_bg_d, 0, nullptr, 0.0f, N, b.S, 1, lr, F(b.z_c_comp), st))) return rc;
        if ((rc = outside(F(b.z_c), b.S, 1, F(b.xyz_c), F(b.dreal_c)))) return rc;
        bo.rgb = F(p.rgb_b);
        bo.depth = o.depth ? F(p.depth_b) : nullptr;
        bo.rgb_coarse = F(p.rgb_cb);
        if ((rc = two_pass(bg, b, cnt, include_xyz_real ? 7 : 4, F(p.ld_b), u_fine_bg_d, F(p.dirs), 3, bidx, bo, outside))) return rc;
    }

    // ---- foreground pass (rendering.py:82-87, 176-248); bg_lambda of the final type and of the cascade's coarse type
    // (render.py:317: requested iff there is a background)
    mn_render_outputs fo = o;
    fo.bg_lambda = bg ? (o.bg_lambda ? o.bg_lambda : F(p.lam)) : nullptr;
    fo.bg_lambda_coarse = (bg && use_cascade && fine) ? (o.bg_lambda_coarse ? o.bg_lambda_coarse : F(p.lam_c)) : nullptr;
    if ((rc = mn_sample_coarse(ctx, rays_d, bg ? F(p.far_ov) : nullptr, z_steps_d, nullptr, 0.0f, N, p.fg.S, F(p.fg.z_c),
                               F(p.fg.xyz_c), stream)))
        return rc;
    auto from_z = [&](const float* z, int S, int, float* xyz, float*) { return mn_points_from_z(ctx, rays_d, z, N, S, xyz, stream); };
    if ((rc = two_pass(m, p.fg, nullptr, 3, F(p.last_delta), u_fine_d, rays_d + 3, 8, image_indices_d, fo, from_z))) return rc;
    if (!bg) return MN_OK;

    // ---- blend (render.py:320-340): the final type's rgb / depth, and rgb_coarse under cascade with fine samples
    return blend_bg(ctx, o, bo, fo.bg_lambda, fo.bg_lambda_coarse, I(p.pos), N, st);
}

// ---- mn_render_rays_train(_bg): the recording render and its backward ------------------------------------------------------
// The buffers of one network's recording two-pass render over N rays: S coarse samples, F fine draws, Sq (S + F under cascade, else
// F) fine-query samples, `cols` point columns.  The tape holds what the backward reads: the depths as the composite reads them
// (z_c_comp, z_q_comp; with flip - the background pass - the coarse depths reversed and, under cascade, the fine-query depths
// reversed), the raw rows, the raw SH coefficients of an SH head and the two model tapes.  The workspace holds the depths in sample
// order where they differ (z_c, z_q; kNone: the composite's buffer), the points and, with flip, their real depths, the weights, the
// fine draws before sort_cat (z_f; kNone: the fine-query depths) and the model calls' workspace.  The backward workspace holds the
// per-sample gradients and the model backward's workspace.
// A pass masked by an occupancy grid (occ_idx_c != kNone) runs each model call on its queried samples only, compacted: the tape
// also holds each query's compacted sample indices (occ_idx_c / occ_idx_f) and the two queried-row counts (occ_cnt), and the model
// tapes and raw SH coefficients are in compacted order.  The workspace holds the test flags / compacted positions, the block
// counts, the compacted results and the compacted density noise; the backward workspace the compacted result gradients.
struct TrainPassBufs {
    int S, F, Sq, cols, flip;
    size_t z_c_comp, raw_c, z_q_comp, raw_f, mlp_c, mlp_f, tape_c, tape_f, tape_c_bytes, tape_f_bytes;
    size_t z_c, z_q, z_f, xyz_c, dreal_c, w_c, xyz_f, dreal_f, model_ws, model_ws_bytes;
    size_t g_raw_c, g_raw_f, g_mlp_c, g_mlp_f, bwd_ws, bwd_ws_bytes;
    size_t occ_idx_c = kNone, occ_idx_f = kNone, occ_cnt = kNone, occ_pos, occ_blk, occ_out, occ_noise, g_cmp;
};

// tc: the network trains at MN_PREC_TC_F16 (the model tapes and the backward workspace of the tensor-core pass); occ: the pass
// is masked by an occupancy grid
TrainPassBufs carve_train_pass(Carve& tape, Carve& ws, Carve& bwd, const mn_model* net, int64_t N, int S, int F, int use_cascade,
                               bool sh, int cols, bool flip, bool tc, bool occ = false) {
    TrainPassBufs b{};
    b.S = S; b.F = F; b.Sq = use_cascade ? S + F : F; b.cols = cols; b.flip = flip;
    const int64_t Bc = N * S, Bf = N * b.Sq;
    const int out_cols = net->nd.rgb_dim + 1;
    b.z_c_comp = tape((size_t)Bc * 4);
    b.raw_c = tape((size_t)Bc * 16);
    b.z_q_comp = tape((size_t)Bf * 4);
    b.raw_f = tape((size_t)Bf * 16);
    b.mlp_c = sh ? tape((size_t)Bc * out_cols * 4) : kNone;
    b.mlp_f = sh ? tape((size_t)Bf * out_cols * 4) : kNone;
    b.tape_c_bytes = tc ? mn_model_tape_bytes_tc(net, Bc) : mn_model_tape_bytes(net, Bc);
    b.tape_f_bytes = tc ? mn_model_tape_bytes_tc(net, Bf) : mn_model_tape_bytes(net, Bf);
    b.tape_c = tape(b.tape_c_bytes);
    b.tape_f = tape(b.tape_f_bytes);
    b.z_c = flip ? ws((size_t)Bc * 4) : kNone;
    b.z_q = flip && use_cascade ? ws((size_t)Bf * 4) : kNone;
    b.z_f = use_cascade ? ws((size_t)N * F * 4) : kNone;
    b.xyz_c = ws((size_t)Bc * cols * 4);
    b.dreal_c = flip ? ws((size_t)Bc * 4) : kNone;
    b.w_c = ws((size_t)Bc * 4);
    b.xyz_f = ws((size_t)Bf * cols * 4);
    b.dreal_f = flip ? ws((size_t)Bf * 4) : kNone;
    const size_t a = mn_model_workspace_bytes(net, Bc, MN_PREC_FP32), c = mn_model_workspace_bytes(net, Bf, MN_PREC_FP32);
    b.model_ws_bytes = a > c ? a : c;
    b.model_ws = ws(b.model_ws_bytes);
    b.g_raw_c = bwd((size_t)Bc * 16);
    b.g_raw_f = bwd((size_t)Bf * 16);
    b.g_mlp_c = sh ? bwd((size_t)Bc * out_cols * 4) : kNone;
    b.g_mlp_f = sh ? bwd((size_t)Bf * out_cols * 4) : kNone;
    const size_t ba = tc ? mn_model_backward_workspace_bytes_tc(net, Bc) : mn_model_backward_workspace_bytes(net, Bc);
    const size_t bc = tc ? mn_model_backward_workspace_bytes_tc(net, Bf) : mn_model_backward_workspace_bytes(net, Bf);
    b.bwd_ws_bytes = ba > bc ? ba : bc;
    b.bwd_ws = bwd(b.bwd_ws_bytes);
    if (occ) {
        const int64_t rows = Bc > Bf ? Bc : Bf;
        b.occ_idx_c = tape((size_t)Bc * 4);
        b.occ_idx_f = tape((size_t)Bf * 4);
        b.occ_cnt = tape(2 * 4);
        b.occ_pos = ws((size_t)rows * 4);
        b.occ_blk = ws((size_t)mn_cdiv(rows, kCompactBlock) * 4);
        b.occ_out = ws((size_t)rows * 16);
        b.occ_noise = ws((size_t)rows * 4);
        b.g_cmp = bwd((size_t)rows * 16);
    }
    return b;
}

// The recording two-pass render of one network (render.py `_two_pass`) into the tape T and workspace W, from the coarse depths
// and points the caller wrote (b.z_c, b.z_c_comp, b.xyz_c, b.dreal_c): the recording coarse query, one composite for the
// resampling weights and, under cascade, the coarse type's rgb and bg_lambda (the detached composite of the reference computes
// the same weights), resampling, sort_cat under cascade, the fine points, the recording fine query and the final composite.
// live: the device count of the rays that hold data (background pass), or null for all N.  u, noise_c, noise_f: the fine draws
// and the density noise.  dirs / dstride, idx: per ray.  r and fine_points(z, S, flip_pts, xyz, dreal): as two_pass's.
// A pass carved with an occupancy grid queries through `occ` (query_occ of render_impl, recording); counts_out: as there.
template <class Points>
int train_two_pass(mn_ctx* ctx, mn_model* net, int precision, const TrainPassBufs& b, char* T, char* W, int64_t N, const int* live,
                   int use_cascade, int sh_deg, const float* last_delta, const float* u, const float* noise_c, const float* noise_f,
                   const float* dirs, int64_t dstride, const float* idx, const mn_render_outputs& r, Points&& fine_points,
                   cudaStream_t st, const OccGrid* occ = nullptr, int* counts_out = nullptr) {
    auto TF = [&](size_t off) { return off == kNone ? nullptr : reinterpret_cast<float*>(T + off); };
    auto WF = [&](size_t off) { return off == kNone ? nullptr : reinterpret_cast<float*>(W + off); };
    const LiveRows lr{live, 1};
    const bool sh = sh_deg >= 0;
    float* z_c = b.z_c == kNone ? TF(b.z_c_comp) : WF(b.z_c);
    float* z_q = b.z_q == kNone ? TF(b.z_q_comp) : WF(b.z_q);
    float* z_f = b.z_f == kNone ? z_q : WF(b.z_f);

    // one recording model query on [N, S, cols] points -> raw [N, S, 4], into the model tape at `tape` (render.py `_query`)
    auto query = [&](const float* xyz, int S, int coarse, const float* noise, float* mlp_out, float* raw_out, size_t tape,
                     size_t tape_n) -> int {
        mn_rows rows{};
        rows.mode = 1;
        rows.x_d = xyz;
        rows.cols = b.cols;
        rows.dirs_d = net->d.pos_dir_dim > 0 ? dirs : nullptr;
        rows.dir_stride = dstride;
        rows.idx_d = net->d.appearance_dim > 0 ? idx : nullptr;
        rows.samples_per_ray = S;
        const LiveRows lrs{live, S};
        int e = mn_model_forward_train_live(ctx, net, &rows, N * S, lrs, coarse, noise, precision, sh ? mlp_out : raw_out, T + tape,
                                            tape_n, W + b.model_ws, b.model_ws_bytes, st);
        if (e) return e;
        if (sh) return mn_stage_sh_to_rgb(ctx, sh_deg, mlp_out, net->nd.rgb_dim + 1, dirs, dstride, S, N * S, 1, lrs, raw_out, st);
        return MN_OK;
    };
    // The same through the occupancy grid: test and compaction of the N * S samples (their indices and count into the tape at
    // idx_off / b.occ_cnt + pass, each queried sample's noise to its compacted row), the recording model call and the SH head on
    // the compacted rows, then every raw row from them or zero.  pass: 0 coarse, 1 fine.
    auto query_occ = [&](const float* xyz, int S, int coarse, const float* noise, float* mlp_out, float* raw_out, size_t tape,
                         size_t tape_n, size_t idx_off, int pass) -> int {
        const int64_t n = N * S;
        const unsigned nblk = (unsigned)mn_cdiv(n, kCompactBlock);
        int* pos = reinterpret_cast<int*>(W + b.occ_pos);
        int* blk = reinterpret_cast<int*>(W + b.occ_blk);
        int* gather = reinterpret_cast<int*>(T + idx_off);
        int* cnt = reinterpret_cast<int*>(T + b.occ_cnt) + pass;
        float* noise_cmp = noise ? WF(b.occ_noise) : nullptr;
        occ_test_kernel<<<nblk, kCompactBlock, 0, st>>>(xyz, n, *occ, pos, blk);
        MN_LAUNCH_CHECK(ctx);
        occ_compact_kernel<<<nblk, kCompactBlock, 0, st>>>(n, blk, pos, gather, cnt, counts_out ? counts_out + pass : nullptr, noise,
                                                           noise_cmp);
        MN_LAUNCH_CHECK(ctx);
        mn_rows rows{};
        rows.mode = 1;
        rows.x_d = xyz;
        rows.cols = b.cols;
        rows.dirs_d = net->d.pos_dir_dim > 0 ? dirs : nullptr;
        rows.dir_stride = dstride;
        rows.idx_d = net->d.appearance_dim > 0 ? idx : nullptr;
        rows.samples_per_ray = S;
        const LiveRows lrs{cnt, 1};
        float* cmp = WF(b.occ_out);
        int e = mn_model_forward_train_live(ctx, net, &rows, n, lrs, coarse, noise_cmp, precision, sh ? mlp_out : cmp, T + tape, tape_n,
                                            W + b.model_ws, b.model_ws_bytes, st, gather);
        if (e) return e;
        if (sh && (e = mn_stage_sh_to_rgb(ctx, sh_deg, mlp_out, net->nd.rgb_dim + 1, dirs, dstride, S, n, 1, lrs, cmp, st, gather)))
            return e;
        occ_scatter_kernel<<<(unsigned)mn_cdiv(n, 256), 256, 0, st>>>(reinterpret_cast<const float4*>(cmp), pos, n,
                                                                      reinterpret_cast<float4*>(raw_out));
        MN_LAUNCH_CHECK(ctx);
        return MN_OK;
    };
    const bool masked = b.occ_idx_c != kNone;

    int rc;
    if (masked) rc = query_occ(WF(b.xyz_c), b.S, 1, noise_c, TF(b.mlp_c), TF(b.raw_c), b.tape_c, b.tape_c_bytes, b.occ_idx_c, 0);
    else rc = query(WF(b.xyz_c), b.S, 1, noise_c, TF(b.mlp_c), TF(b.raw_c), b.tape_c, b.tape_c_bytes);
    if (rc) return rc;
    if ((rc = mn_stage_composite(ctx, TF(b.raw_c), TF(b.z_c_comp), WF(b.dreal_c), b.S, nullptr, nullptr, nullptr, 0, last_delta, N,
                                 b.flip, lr, WF(b.w_c), use_cascade ? r.rgb_coarse : nullptr, nullptr, nullptr,
                                 use_cascade ? r.bg_lambda_coarse : nullptr, st)))
        return rc;
    if ((rc = mn_stage_sample_pdf(ctx, z_c, WF(b.w_c), b.S, nullptr, u, b.F, N, b.S, b.F, lr, z_f, nullptr, nullptr, st))) return rc;
    if (use_cascade)
        if ((rc = mn_stage_sort_cat(ctx, z_c, b.S, z_f, b.F, N, 0, lr, z_q, b.flip ? TF(b.z_q_comp) : nullptr, st))) return rc;
    if ((rc = fine_points(z_q, b.Sq, b.flip && use_cascade, WF(b.xyz_f), WF(b.dreal_f)))) return rc;
    if (masked) rc = query_occ(WF(b.xyz_f), b.Sq, 0, noise_f, TF(b.mlp_f), TF(b.raw_f), b.tape_f, b.tape_f_bytes, b.occ_idx_f, 1);
    else rc = query(WF(b.xyz_f), b.Sq, 0, noise_f, TF(b.mlp_f), TF(b.raw_f), b.tape_f, b.tape_f_bytes);
    if (rc) return rc;
    // depth scratch when only the variance is wanted: the coarse weights are dead by now
    float* depth = r.depth ? r.depth : (r.depth_var ? WF(b.w_c) : nullptr);
    if (use_cascade)
        return mn_stage_composite(ctx, TF(b.raw_f), TF(b.z_q_comp), WF(b.dreal_f), b.Sq, nullptr, nullptr, nullptr, 0, last_delta, N,
                                  b.flip, lr, nullptr, r.rgb, depth, r.depth_var, r.bg_lambda, st);
    return mn_stage_composite(ctx, TF(b.raw_f), TF(b.z_q_comp), WF(b.dreal_f), b.Sq, TF(b.raw_c), TF(b.z_c_comp), WF(b.dreal_c), b.S,
                              last_delta, N, b.flip, lr, nullptr, r.rgb, depth, r.depth_var, r.bg_lambda, st);
}

// The result gradients of the queried samples in compacted order: g_cmp[p] = g_raw[idx[p]] for the *count queried rows.
__global__ void occ_gather_grad_kernel(const float4* __restrict__ g_raw, const int* __restrict__ idx, const int* __restrict__ count,
                                       float4* __restrict__ g_cmp) {
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= *count) return;
    g_cmp[p] = g_raw[idx[p]];
}

// The backward of train_two_pass: the composite backward(s) - with the gradients of bg_lambda (g_lam, g_lam_c; null: none) - then
// the fine and the coarse model backwards, each through the SH head's backward, into gw.  The coarse pass has no gradient under
// cascade without g_rgb_coarse, and is skipped.  dirs / dstride: the directions the forward read.  A pass masked by an occupancy
// grid gathers the per-sample gradients of its queried samples into compacted order first (occ_gather_grad_kernel) and runs the
// SH head's and the model's backward over the queried rows only; a skipped sample's gradient reaches no parameter.
int train_two_pass_backward(mn_ctx* ctx, mn_model* net, int precision, const TrainPassBufs& b, const char* T, char* W, int64_t N,
                            const int* live, int use_cascade, int sh_deg, const float* last_delta, const float* dirs, int64_t dstride,
                            const float* g_rgb, const float* g_rgb_coarse, const float* g_lam, const float* g_lam_c, float* gw,
                            cudaStream_t st) {
    auto TF = [&](size_t off) { return off == kNone ? nullptr : reinterpret_cast<const float*>(T + off); };
    auto WF = [&](size_t off) { return off == kNone ? nullptr : reinterpret_cast<float*>(W + off); };
    const LiveRows lr{live, 1};
    const bool coarse = !use_cascade || g_rgb_coarse;
    int rc;

    // composites: the fine one (with the coarse samples merged in, without cascade), the cascade's coarse one
    if (use_cascade) {
        if ((rc = mn_stage_composite_backward(ctx, TF(b.raw_f), TF(b.z_q_comp), b.Sq, nullptr, nullptr, 0, last_delta, N, b.flip, lr,
                                              g_rgb, g_lam, WF(b.g_raw_f), nullptr, st)))
            return rc;
        if (coarse && (rc = mn_stage_composite_backward(ctx, TF(b.raw_c), TF(b.z_c_comp), b.S, nullptr, nullptr, 0, last_delta, N,
                                                        b.flip, lr, g_rgb_coarse, g_lam_c, WF(b.g_raw_c), nullptr, st)))
            return rc;
    } else if ((rc = mn_stage_composite_backward(ctx, TF(b.raw_f), TF(b.z_q_comp), b.Sq, TF(b.raw_c), TF(b.z_c_comp), b.S, last_delta,
                                                 N, b.flip, lr, g_rgb, g_lam, WF(b.g_raw_f), WF(b.g_raw_c), st))) {
        return rc;
    }
    // the model backwards in reverse order of their forward calls, each through the SH head's backward first
    const bool masked = b.occ_idx_c != kNone;
    auto model_bwd = [&](int S, int use_coarse, size_t mlp, size_t g_raw, size_t g_mlp, size_t tape, size_t tape_n, size_t idx_off,
                         int pass) -> int {
        LiveRows lrs{live, S};
        const float* g = WF(g_raw);
        const int* gather = nullptr;
        if (masked) {
            gather = reinterpret_cast<const int*>(T + idx_off);
            lrs = LiveRows{reinterpret_cast<const int*>(T + b.occ_cnt) + pass, 1};
            occ_gather_grad_kernel<<<(unsigned)mn_cdiv(N * S, 256), 256, 0, st>>>(reinterpret_cast<const float4*>(g), gather, lrs.rays,
                                                                                 reinterpret_cast<float4*>(WF(b.g_cmp)));
            MN_LAUNCH_CHECK(ctx);
            g = WF(b.g_cmp);
        }
        int e;
        if (sh_deg >= 0) {
            if ((e = mn_stage_sh_to_rgb_backward(ctx, sh_deg, TF(mlp), net->nd.rgb_dim + 1, dirs, dstride, S, N * S, 1, lrs, g, WF(g_mlp),
                                                 st, gather)))
                return e;
            g = WF(g_mlp);
        }
        return mn_model_backward_live(ctx, net, N * S, lrs, use_coarse, precision, g, T + tape, tape_n, gw, W + b.bwd_ws,
                                      b.bwd_ws_bytes, st);
    };
    if ((rc = model_bwd(b.Sq, 0, b.mlp_f, b.g_raw_f, b.g_mlp_f, b.tape_f, b.tape_f_bytes, b.occ_idx_f, 1))) return rc;
    if (coarse) return model_bwd(b.S, 1, b.mlp_c, b.g_raw_c, b.g_mlp_c, b.tape_c, b.tape_c_bytes, b.occ_idx_c, 0);
    return MN_OK;
}

// mn_render_rays_train: the foreground's pass, and in the tape its last deltas and, for an SH head, a copy of the rays (the
// directions the backward reads).
struct TrainPlan {
    TrainPassBufs pass;
    size_t last_delta, rays, tape_total, ws_total, bwd_total;
};

TrainPlan make_train_plan(const mn_model* m, int64_t N, int S, int F, int use_cascade, bool sh, bool tc, bool occ = false) {
    TrainPlan p{};
    Carve t, w, b;
    p.last_delta = t((size_t)N * 4);
    p.pass = carve_train_pass(t, w, b, m, N, S, F, use_cascade, sh, 3, false, tc, occ);
    p.rays = sh ? t((size_t)N * 32) : kNone;
    p.tape_total = t.off + 256;
    p.ws_total = w.off + 256;
    p.bwd_total = b.off + 256;
    return p;
}

// The checks shared by the train render, its backward and their size queries: a foreground network that trains at `precision`.
int check_train(mn_ctx* ctx, const mn_model* m, int64_t N, int coarse_samples, int fine_samples, int precision, const char* name) {
    const std::string n(name);
    if (N < 0 || coarse_samples < 3 || fine_samples < 1)
        return mn_fail(ctx, MN_ERR_INVALID, n + ": needs N >= 0, >= 3 coarse samples (resampling) and fine_samples > 0");
    if (precision != MN_PREC_FP32 && precision != MN_PREC_TC_F16)
        return mn_fail(ctx, MN_ERR_INVALID, n + ": training precision is MN_PREC_FP32 or MN_PREC_TC_F16");
    if (precision == MN_PREC_TC_F16 && !mn_model_train_tc_supported(m)) return mn_fail(ctx, MN_ERR_UNSUPPORTED, MN_TC_TRAIN_COVERAGE);
    return MN_OK;
}

// The checks of a training render through an occupancy grid (those of render_impl), and the grid as the kernels read it.
int check_occ(mn_ctx* ctx, const mn_occupancy* occ, int64_t N, int S, int F, int use_cascade, const char* name, OccGrid* g) {
    const std::string n(name);
    if (!occ->bits || occ->reso < 1 || occ->reso > MN_OCC_MAX_RESO)
        return mn_fail(ctx, MN_ERR_INVALID, n + ": the occupancy grid needs bits and a reso of 1.." + std::to_string(MN_OCC_MAX_RESO));
    const int Sq = use_cascade ? S + F : F;
    if (N * (int64_t)(Sq > S ? Sq : S) > INT32_MAX)
        return mn_fail(ctx, MN_ERR_INVALID, n + ": an occupancy-grid render indexes at most 2^31 - 1 samples per pass");
    g->bits = occ->bits;
    g->reso = occ->reso;
    for (int a = 0; a < 3; ++a) { g->off[a] = occ->offset[a]; g->scl[a] = occ->scale[a]; }
    return MN_OK;
}

int train_impl(mn_ctx* ctx, mn_model* m, const float* rays_d, const float* image_indices_d, int64_t N, const float* z_steps_d,
               const float* jitter_d, float perturb, int S, const float* noise_c_d, const float* u_d, const float* noise_f_d, int F,
               int use_cascade, int sh_deg, int precision, float* rgb, float* depth, float* var, float* rgb_coarse, void* tape_d,
               size_t tape_bytes, void* workspace_d, size_t workspace_bytes, cudaStream_t st, const char* name,
               const mn_occupancy* occ = nullptr, int* counts_out = nullptr) {
    const std::string nm(name);
    if (!ctx || !m || !rays_d || !z_steps_d || !u_d || !rgb) return MN_ERR_INVALID;
    int rc;
    if ((rc = check_train(ctx, m, N, S, F, precision, name))) return rc;
    if ((rc = check_net(ctx, m, use_cascade, F, sh_deg, image_indices_d, name))) return rc;
    if (perturb > 0 && !jitter_d) return mn_fail(ctx, MN_ERR_INVALID, nm + ": perturb > 0 needs jitter_d");
    if (use_cascade && !rgb_coarse) return mn_fail(ctx, MN_ERR_INVALID, nm + ": rgb_coarse_out_d is required under use_cascade");
    OccGrid G{};
    if (occ && (rc = check_occ(ctx, occ, N, S, F, use_cascade, name, &G))) return rc;
    if (N == 0) return MN_OK;
    const TrainPlan p = make_train_plan(m, N, S, F, use_cascade, sh_deg >= 0, precision == MN_PREC_TC_F16, occ != nullptr);
    if (!tape_d || tape_bytes < p.tape_total) return mn_fail(ctx, MN_ERR_WORKSPACE, nm + ": tape too small");
    if (!workspace_d || workspace_bytes < p.ws_total) return mn_fail(ctx, MN_ERR_WORKSPACE, nm + ": workspace too small");
    char* T = (char*)tape_d;
    char* W = (char*)workspace_d;
    float* last_delta = reinterpret_cast<float*>(T + p.last_delta);
    fill_kernel<<<(unsigned)mn_cdiv(N, 256), 256, 0, st>>>(last_delta, N, 1e10f);   // rendering.py:33
    MN_LAUNCH_CHECK(ctx);
    if (p.rays != kNone) MN_CUDA(ctx, cudaMemcpyAsync(T + p.rays, rays_d, (size_t)N * 32, cudaMemcpyDeviceToDevice, st));
    if ((rc = mn_sample_coarse(ctx, rays_d, nullptr, z_steps_d, jitter_d, perturb, N, S, reinterpret_cast<float*>(T + p.pass.z_c_comp),
                               reinterpret_cast<float*>(W + p.pass.xyz_c), st)))
        return rc;
    mn_render_outputs o{};
    o.rgb = rgb;
    o.depth = depth;
    o.depth_var = var;
    o.rgb_coarse = rgb_coarse;
    auto from_z = [&](const float* z, int Sq, int, float* xyz, float*) { return mn_points_from_z(ctx, rays_d, z, N, Sq, xyz, st); };
    return train_two_pass(ctx, m, precision, p.pass, T, W, N, nullptr, use_cascade, sh_deg, last_delta, u_d, noise_c_d, noise_f_d,
                          rays_d + 3, 8, image_indices_d, o, from_z, st, occ ? &G : nullptr, counts_out);
}

int train_backward_impl(mn_ctx* ctx, mn_model* m, int64_t N, int S, int F, int use_cascade, int sh_deg, int precision,
                        const float* g_rgb, const float* g_rgb_coarse, const void* tape_d, size_t tape_bytes, float* gw,
                        void* workspace_d, size_t workspace_bytes, cudaStream_t st, const char* name, bool occ = false) {
    const std::string nm(name);
    if (!ctx || !m || !g_rgb || !gw) return MN_ERR_INVALID;
    int rc;
    if ((rc = check_train(ctx, m, N, S, F, precision, name))) return rc;
    if (N == 0) return MN_OK;
    const TrainPlan p = make_train_plan(m, N, S, F, use_cascade, sh_deg >= 0, precision == MN_PREC_TC_F16, occ);
    if (!tape_d || tape_bytes < p.tape_total) return mn_fail(ctx, MN_ERR_WORKSPACE, nm + ": tape too small");
    if (!workspace_d || workspace_bytes < p.bwd_total) return mn_fail(ctx, MN_ERR_WORKSPACE, nm + ": workspace too small");
    const char* T = (const char*)tape_d;
    const float* dirs = p.rays == kNone ? nullptr : reinterpret_cast<const float*>(T + p.rays) + 3;
    return train_two_pass_backward(ctx, m, precision, p.pass, T, (char*)workspace_d, N, nullptr, use_cascade, sh_deg,
                                   reinterpret_cast<const float*>(T + p.last_delta), dirs, 8, g_rgb, g_rgb_coarse, nullptr, nullptr, gw,
                                   st);
}

// ---- mn_render_rays_train_bg: the recording render with a background network and its backward ------------------------------
// Rows of a [N, cols] draw block of ray ids -> its rows in compacted order: dst[p] = src[ids[p]] for the live background rays.
__global__ void gather_rows_kernel(const float* __restrict__ src, const int64_t* __restrict__ ids, const int* __restrict__ count,
                                   int64_t N, int cols, float* __restrict__ dst) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (int64_t)*count * cols) return;
    const int64_t p = t / cols;
    dst[t] = src[ids[p] * cols + (t - p * cols)];
}

// torch.flip(z, [-1]) of the live rows of [N, S]
__global__ void flip_rows_kernel(const float* __restrict__ z, int64_t N, int S, LiveRows live, float* __restrict__ out) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= live.rows(N) * S) return;
    const int64_t r = t / S;
    out[r * S + (S - 1 - (t - r * S))] = z[t];
}

// Backward of the lambda blend val + bg_val[pos] * lam (bg_blend_kernel, torch's mul and index backwards): g_bg[pos[i]] =
// g[i] * lam[i]; g_lam[i] = sum_c g[i, c] * bg_val[pos[i], c], 0 for a ray that stays in the foreground.
__global__ void bg_blend_backward_kernel(const float* __restrict__ g, const float* __restrict__ lam, const float* __restrict__ bg_val,
                                         const int* __restrict__ pos, int64_t N, float* __restrict__ g_lam, float* __restrict__ g_bg) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const int p = pos[i];
    float gl = 0.0f;
    if (p >= 0) {
        const float* gi = g + i * 3;
        const float* b = bg_val + (int64_t)p * 3;
        for (int c = 0; c < 3; ++c) g_bg[(int64_t)p * 3 + c] = __fmul_rn(gi[c], lam[i]);
        gl = __fadd_rn(__fadd_rn(__fmul_rn(gi[0], b[0]), __fmul_rn(gi[1], b[1])), __fmul_rn(gi[2], b[2]));
    }
    g_lam[i] = gl;
}

// The buffers of the recording render with a background network over N rays (the compacted background rays first), after the
// foreground's TrainPlan in each of the three regions, then the background network's pass (half the foreground's samples).  Tape:
// the split (compacted positions and count), the background's last deltas, the blend's inputs (bg_lambda of both types, the
// background colours) and the compacted directions.  Workspace: the rest of the split (far override, block counts, ids, image
// indices), the background depth and the gathered draws of ray-indexed blocks.  Backward workspace: the blend's gradients.
struct BgTrainPlan {
    TrainPlan fg;
    TrainPassBufs bg;
    size_t pos, count, ld_b, lam, lam_c, rgb_b, rgb_cb, dirs, tape_total;
    size_t far_ov, blk, ids, idx, depth_b, jit, u, noise_c, noise_f, ws_total;
    size_t g_rgb_b, g_rgb_cb, g_lam, g_lam_c, bwd_total;
};

BgTrainPlan make_bg_train_plan(const mn_model* m, const mn_model* bg, int64_t N, int Sc, int Sf, int use_cascade, bool sh, bool tc,
                               bool bg_tc, bool occ = false) {
    BgTrainPlan p{};
    p.fg = make_train_plan(m, N, Sc, Sf, use_cascade, sh, tc, occ);
    Carve t, w, b;
    t.off = p.fg.tape_total;
    w.off = p.fg.ws_total;
    b.off = p.fg.bwd_total;
    p.pos = t((size_t)N * 4);
    p.count = t(4);
    p.ld_b = t((size_t)N * 4);
    p.lam = t((size_t)N * 4);
    p.lam_c = t((size_t)N * 4);
    p.rgb_b = t((size_t)N * 12);
    p.rgb_cb = t((size_t)N * 12);
    p.dirs = t((size_t)N * 12);
    p.far_ov = w((size_t)N * 4);
    p.blk = w((size_t)mn_cdiv(N, kCompactBlock) * 4);
    p.ids = w((size_t)N * 8);
    p.idx = w((size_t)N * 4);
    p.g_rgb_b = b((size_t)N * 12);
    p.g_rgb_cb = b((size_t)N * 12);
    p.g_lam = b((size_t)N * 4);
    p.g_lam_c = b((size_t)N * 4);
    // the real-xyz routing prefix, then [point, 1/r]
    p.bg = carve_train_pass(t, w, b, bg, N, Sc / 2, Sf / 2, use_cascade, sh, bg->d.kind == 2 && bg->d.xyz_real ? 7 : 4, true, bg_tc);
    p.depth_b = w((size_t)N * 4);
    p.jit = w((size_t)N * p.bg.S * 4);
    p.u = w((size_t)N * p.bg.F * 4);
    p.noise_c = w((size_t)N * p.bg.S * 4);
    p.noise_f = w((size_t)N * p.bg.Sq * 4);
    p.tape_total = t.off + 256;
    p.ws_total = w.off + 256;
    p.bwd_total = b.off + 256;
    return p;
}

// The checks shared by the background train render, its backward and their size queries.
int check_train_bg(mn_ctx* ctx, const mn_model* m, const mn_model* bg, int64_t N, int Sc, int Sf, int precision, int bg_precision,
                   const char* name) {
    int rc;
    if ((rc = check_train(ctx, m, N, Sc, Sf, precision, name))) return rc;
    if ((rc = check_train(ctx, bg, N, Sc / 2, Sf / 2, bg_precision, name))) return rc;
    return MN_OK;
}

int train_bg_impl(mn_ctx* ctx, mn_model* m, mn_model* bg, const float* rays_d, const float* image_indices_d, int64_t N,
                  const float* center_d, const float* radius_d, int include_xyz_real, int cluster_2d, const float* z_steps_d,
                  const float* z_steps_bg_d, const float* jitter_d, const float* jitter_bg_d, float perturb, int Sc,
                  const float* noise_c_d, const float* noise_c_bg_d, const float* u_d, const float* u_bg_d, const float* noise_f_d,
                  const float* noise_f_bg_d, int Sf, int use_cascade, int sh_deg, int precision, int bg_precision, int by_ray,
                  const mn_render_outputs* out, void* tape_d, size_t tape_bytes, void* workspace_d, size_t workspace_bytes,
                  cudaStream_t st, const char* name, const mn_occupancy* occ = nullptr, int* counts_out = nullptr) {
    const std::string nm(name);
    if (!ctx || !m || !bg || !rays_d || !z_steps_d || !z_steps_bg_d || !u_d || !u_bg_d || !out || !out->rgb || !out->bg_lambda)
        return MN_ERR_INVALID;
    const mn_render_outputs& o = *out;
    int rc;
    if ((rc = check_train_bg(ctx, m, bg, N, Sc, Sf, precision, bg_precision, name))) return rc;
    if ((rc = check_net(ctx, m, use_cascade, Sf, sh_deg, image_indices_d, name))) return rc;
    if ((rc = check_net(ctx, bg, use_cascade, Sf, sh_deg, image_indices_d, name))) return rc;
    if (perturb > 0 && (!jitter_d || !jitter_bg_d)) return mn_fail(ctx, MN_ERR_INVALID, nm + ": perturb > 0 needs jitter_d and jitter_bg_d");
    if (use_cascade && (!o.rgb_coarse || !o.bg_lambda_coarse))
        return mn_fail(ctx, MN_ERR_INVALID, nm + ": rgb_coarse and bg_lambda_coarse are required under use_cascade");
    if (radius_d && !center_d) return mn_fail(ctx, MN_ERR_INVALID, nm + ": sphere radius without a center");
    if (include_xyz_real != (bg->d.kind == 2 && bg->d.xyz_real ? 1 : 0))
        return mn_fail(ctx, MN_ERR_INVALID, nm + ": include_xyz_real must match the background model's real-xyz prefix");
    OccGrid G{};
    if (occ && (rc = check_occ(ctx, occ, N, Sc, Sf, use_cascade, name, &G))) return rc;
    if (N == 0) return MN_OK;
    const BgTrainPlan p = make_bg_train_plan(m, bg, N, Sc, Sf, use_cascade, sh_deg >= 0, precision == MN_PREC_TC_F16,
                                             bg_precision == MN_PREC_TC_F16, occ != nullptr);
    if (!tape_d || tape_bytes < p.tape_total) return mn_fail(ctx, MN_ERR_WORKSPACE, nm + ": tape too small");
    if (!workspace_d || workspace_bytes < p.ws_total) return mn_fail(ctx, MN_ERR_WORKSPACE, nm + ": workspace too small");
    char* T = (char*)tape_d;
    char* W = (char*)workspace_d;
    auto TF = [&](size_t off) { return reinterpret_cast<float*>(T + off); };
    auto WF = [&](size_t off) { return reinterpret_cast<float*>(W + off); };
    int* pos = reinterpret_cast<int*>(T + p.pos);
    int* cnt = reinterpret_cast<int*>(T + p.count);
    int64_t* ids = reinterpret_cast<int64_t*>(W + p.ids);
    const LiveRows lr{cnt, 1};
    const TrainPassBufs& b = p.bg;

    // ---- split and compaction (render.py:327-342): the foreground's last deltas land in its tape
    float* bidx = image_indices_d ? WF(p.idx) : nullptr;
    if ((rc = split_bg(ctx, rays_d, image_indices_d, N, center_d, radius_d, WF(p.far_ov), TF(p.fg.last_delta), pos,
                       reinterpret_cast<int*>(W + p.blk), cnt, ids, TF(p.dirs), bidx, TF(p.ld_b), st)))
        return rc;

    // ---- the background draws in compacted order: ray-indexed blocks are gathered at the background rays
    const float *jit = jitter_bg_d, *ub = u_bg_d, *nc = noise_c_bg_d, *nf = noise_f_bg_d;
    if (by_ray) {
        auto gather = [&](const float*& src, int cols, size_t dst) -> int {
            if (!src) return MN_OK;
            gather_rows_kernel<<<(unsigned)mn_cdiv(N * cols, 256), 256, 0, st>>>(src, ids, cnt, N, cols, WF(dst));
            MN_LAUNCH_CHECK(ctx);
            src = WF(dst);
            return MN_OK;
        };
        if ((rc = gather(jit, b.S, p.jit)) || (rc = gather(ub, b.F, p.u)) || (rc = gather(nc, b.S, p.noise_c)) ||
            (rc = gather(nf, b.Sq, p.noise_f)))
            return rc;
    }

    // ---- background pass over the compacted rays (render.py `bg_pass`, `_two_pass` flipped): stratified depths in sample order
    // and reversed, the points outside the sphere in reversed sample order
    auto outside = [&](const float* z, int S, int flip_pts, float* xyz, float* dreal) {
        return mn_stage_points_outside(ctx, rays_d, ids, z, center_d, radius_d, N, S, include_xyz_real, cluster_2d, flip_pts, lr, xyz,
                                       dreal, st);
    };
    if ((rc = mn_stage_stratify(ctx, z_steps_bg_d, 0, jit, perturb, N, b.S, 0, lr, WF(b.z_c), st))) return rc;
    flip_rows_kernel<<<(unsigned)mn_cdiv(N * b.S, 256), 256, 0, st>>>(WF(b.z_c), N, b.S, lr, TF(b.z_c_comp));
    MN_LAUNCH_CHECK(ctx);
    if ((rc = outside(WF(b.z_c), b.S, 1, WF(b.xyz_c), WF(b.dreal_c)))) return rc;
    mn_render_outputs bo{};
    bo.rgb = TF(p.rgb_b);
    bo.depth = o.depth ? WF(p.depth_b) : nullptr;
    bo.rgb_coarse = TF(p.rgb_cb);
    if ((rc = train_two_pass(ctx, bg, bg_precision, b, T, W, N, cnt, use_cascade, sh_deg, TF(p.ld_b), ub, nc, nf, TF(p.dirs), 3, bidx,
                             bo, outside, st)))
        return rc;

    // ---- foreground pass with the far override, the last deltas and bg_lambda of both types (render.py:344-348)
    mn_render_outputs fo = o;
    fo.bg_lambda = TF(p.lam);
    fo.bg_lambda_coarse = use_cascade ? TF(p.lam_c) : nullptr;
    if (p.fg.rays != kNone) MN_CUDA(ctx, cudaMemcpyAsync(T + p.fg.rays, rays_d, (size_t)N * 32, cudaMemcpyDeviceToDevice, st));
    if ((rc = mn_sample_coarse(ctx, rays_d, WF(p.far_ov), z_steps_d, jitter_d, perturb, N, Sc, TF(p.fg.pass.z_c_comp),
                               WF(p.fg.pass.xyz_c), st)))
        return rc;
    auto from_z = [&](const float* z, int Sq, int, float* xyz, float*) { return mn_points_from_z(ctx, rays_d, z, N, Sq, xyz, st); };
    if ((rc = train_two_pass(ctx, m, precision, p.fg.pass, T, W, N, nullptr, use_cascade, sh_deg, TF(p.fg.last_delta), u_d, noise_c_d,
                             noise_f_d, rays_d + 3, 8, image_indices_d, fo, from_z, st, occ ? &G : nullptr, counts_out)))
        return rc;
    MN_CUDA(ctx, cudaMemcpyAsync(o.bg_lambda, fo.bg_lambda, (size_t)N * 4, cudaMemcpyDeviceToDevice, st));
    if (use_cascade) MN_CUDA(ctx, cudaMemcpyAsync(o.bg_lambda_coarse, fo.bg_lambda_coarse, (size_t)N * 4, cudaMemcpyDeviceToDevice, st));

    // ---- blend (render.py:350-376)
    return blend_bg(ctx, o, bo, fo.bg_lambda, fo.bg_lambda_coarse, pos, N, st);
}

int train_bg_backward_impl(mn_ctx* ctx, mn_model* m, mn_model* bg, int64_t N, int Sc, int Sf, int use_cascade, int sh_deg, int precision,
                           int bg_precision, const float* g_rgb, const float* g_rgb_coarse, const void* tape_d, size_t tape_bytes,
                           float* gw, float* gw_bg, void* workspace_d, size_t workspace_bytes, cudaStream_t st, const char* name,
                           bool occ = false) {
    const std::string nm(name);
    if (!ctx || !m || !bg || !g_rgb || !gw || !gw_bg) return MN_ERR_INVALID;
    int rc;
    if ((rc = check_train_bg(ctx, m, bg, N, Sc, Sf, precision, bg_precision, name))) return rc;
    if (N == 0) return MN_OK;
    const BgTrainPlan p = make_bg_train_plan(m, bg, N, Sc, Sf, use_cascade, sh_deg >= 0, precision == MN_PREC_TC_F16,
                                             bg_precision == MN_PREC_TC_F16, occ);
    if (!tape_d || tape_bytes < p.tape_total) return mn_fail(ctx, MN_ERR_WORKSPACE, nm + ": tape too small");
    if (!workspace_d || workspace_bytes < p.bwd_total) return mn_fail(ctx, MN_ERR_WORKSPACE, nm + ": workspace too small");
    const char* T = (const char*)tape_d;
    char* W = (char*)workspace_d;
    auto TF = [&](size_t off) { return reinterpret_cast<const float*>(T + off); };
    auto WF = [&](size_t off) { return reinterpret_cast<float*>(W + off); };
    const int* pos = reinterpret_cast<const int*>(T + p.pos);
    const bool coarse = use_cascade && g_rgb_coarse;      // the cascade's coarse type has a gradient

    // ---- blend backward: the background colours' and bg_lambda's gradients
    auto blend_bwd = [&](const float* g, size_t lam, size_t bval, size_t g_lam, size_t g_bg) -> int {
        bg_blend_backward_kernel<<<(unsigned)mn_cdiv(N, 256), 256, 0, st>>>(g, TF(lam), TF(bval), pos, N, WF(g_lam), WF(g_bg));
        MN_LAUNCH_CHECK(ctx);
        return MN_OK;
    };
    if ((rc = blend_bwd(g_rgb, p.lam, p.rgb_b, p.g_lam, p.g_rgb_b))) return rc;
    if (coarse && (rc = blend_bwd(g_rgb_coarse, p.lam_c, p.rgb_cb, p.g_lam_c, p.g_rgb_cb))) return rc;

    // ---- foreground: composites (with bg_lambda) and model backwards
    const float* dirs = p.fg.rays == kNone ? nullptr : TF(p.fg.rays) + 3;
    if ((rc = train_two_pass_backward(ctx, m, precision, p.fg.pass, T, W, N, nullptr, use_cascade, sh_deg, TF(p.fg.last_delta), dirs, 8,
                                      g_rgb, g_rgb_coarse, WF(p.g_lam), coarse ? WF(p.g_lam_c) : nullptr, gw, st)))
        return rc;

    // ---- background: composites, then the model backwards over the live rows
    return train_two_pass_backward(ctx, bg, bg_precision, p.bg, T, W, N, reinterpret_cast<const int*>(T + p.count), use_cascade, sh_deg,
                                   TF(p.ld_b), TF(p.dirs), 3, WF(p.g_rgb_b), coarse ? WF(p.g_rgb_cb) : nullptr, nullptr, nullptr,
                                   gw_bg, st);
}

}  // namespace

extern "C" {

size_t mn_render_rays_workspace_bytes(const mn_model* m, int64_t N, int coarse_samples, int fine_samples, int use_cascade,
                                      int sh_deg, int precision) {
    if (!m || N < 0 || coarse_samples < 1 || fine_samples < 0) return 0;
    return make_plan(m, nullptr, N, coarse_samples, fine_samples, use_cascade, sh_deg >= 0, precision).total;
}

int mn_render_rays(mn_ctx* ctx, mn_model* m, const float* rays_d, const float* image_indices_d, int64_t N,
                   const float* z_steps_d, int coarse_samples, const float* u_fine_d, int fine_samples, int use_cascade,
                   int sh_deg, int precision, float* rgb_out_d, float* depth_out_d, float* depth_var_out_d,
                   float* rgb_coarse_out_d, void* workspace_d, size_t workspace_bytes, void* stream) {
    mn_render_outputs o{};
    o.rgb = rgb_out_d;
    o.depth = depth_out_d;
    o.depth_var = depth_var_out_d;
    o.rgb_coarse = rgb_coarse_out_d;
    return render_impl(ctx, m, nullptr, rays_d, image_indices_d, N, nullptr, nullptr, 0, 0, z_steps_d, nullptr, coarse_samples,
                       u_fine_d, nullptr, fine_samples, use_cascade, sh_deg, precision, o, workspace_d, workspace_bytes, stream,
                       "mn_render_rays");
}

size_t mn_render_rays_bg_workspace_bytes(const mn_model* fg, const mn_model* bg, int64_t N, int coarse_samples, int fine_samples,
                                         int use_cascade, int sh_deg, int precision) {
    if (!fg || !bg || N < 0 || coarse_samples < 1 || fine_samples < 0) return 0;
    return make_plan(fg, bg, N, coarse_samples, fine_samples, use_cascade, sh_deg >= 0, precision).total;
}

int mn_render_rays_bg(mn_ctx* ctx, mn_model* fg, mn_model* bg, const float* rays_d, const float* image_indices_d, int64_t N,
                      const float* sphere_center3_d, const float* sphere_radius3_d, int include_xyz_real, int cluster_2d,
                      const float* z_steps_d, const float* z_steps_bg_d, int coarse_samples, const float* u_fine_d,
                      const float* u_fine_bg_d, int fine_samples, int use_cascade, int sh_deg, int precision,
                      const mn_render_outputs* out, void* workspace_d, size_t workspace_bytes, void* stream) {
    if (!out) return MN_ERR_INVALID;
    return render_impl(ctx, fg, bg, rays_d, image_indices_d, N, sphere_center3_d, sphere_radius3_d, include_xyz_real, cluster_2d,
                       z_steps_d, z_steps_bg_d, coarse_samples, u_fine_d, u_fine_bg_d, fine_samples, use_cascade, sh_deg, precision,
                       *out, workspace_d, workspace_bytes, stream, bg ? "mn_render_rays_bg" : "mn_render_rays");
}

size_t mn_render_rays_occ_workspace_bytes(const mn_model* m, int64_t N, int coarse_samples, int fine_samples, int use_cascade,
                                          int sh_deg, int precision) {
    if (!m || N < 0 || coarse_samples < 1 || fine_samples < 0) return 0;
    return make_plan(m, nullptr, N, coarse_samples, fine_samples, use_cascade, sh_deg >= 0, precision, true).total;
}

int mn_render_rays_occ(mn_ctx* ctx, mn_model* m, const float* rays_d, const float* image_indices_d, int64_t N,
                       const float* z_steps_d, int coarse_samples, const float* u_fine_d, int fine_samples, int use_cascade,
                       int sh_deg, int precision, const mn_occupancy* occ, int32_t* counts_out_d, float* rgb_out_d,
                       float* depth_out_d, float* depth_var_out_d, float* rgb_coarse_out_d, void* workspace_d,
                       size_t workspace_bytes, void* stream) {
    if (!occ) return mn_fail(ctx, MN_ERR_INVALID, "mn_render_rays_occ: occ is NULL");
    mn_render_outputs o{};
    o.rgb = rgb_out_d;
    o.depth = depth_out_d;
    o.depth_var = depth_var_out_d;
    o.rgb_coarse = rgb_coarse_out_d;
    return render_impl(ctx, m, nullptr, rays_d, image_indices_d, N, nullptr, nullptr, 0, 0, z_steps_d, nullptr, coarse_samples,
                       u_fine_d, nullptr, fine_samples, use_cascade, sh_deg, precision, o, workspace_d, workspace_bytes, stream,
                       "mn_render_rays_occ", occ, counts_out_d);
}

size_t mn_render_rays_bg_occ_workspace_bytes(const mn_model* fg, const mn_model* bg, int64_t N, int coarse_samples, int fine_samples,
                                             int use_cascade, int sh_deg, int precision) {
    if (!fg || !bg || N < 0 || coarse_samples < 1 || fine_samples < 0) return 0;
    return make_plan(fg, bg, N, coarse_samples, fine_samples, use_cascade, sh_deg >= 0, precision, true).total;
}

int mn_render_rays_bg_occ(mn_ctx* ctx, mn_model* fg, mn_model* bg, const float* rays_d, const float* image_indices_d, int64_t N,
                          const float* sphere_center3_d, const float* sphere_radius3_d, int include_xyz_real, int cluster_2d,
                          const float* z_steps_d, const float* z_steps_bg_d, int coarse_samples, const float* u_fine_d,
                          const float* u_fine_bg_d, int fine_samples, int use_cascade, int sh_deg, int precision,
                          const mn_occupancy* occ, int32_t* counts_out_d, const mn_render_outputs* out, void* workspace_d,
                          size_t workspace_bytes, void* stream) {
    if (!out || !bg) return MN_ERR_INVALID;
    if (!occ) return mn_fail(ctx, MN_ERR_INVALID, "mn_render_rays_bg_occ: occ is NULL");
    return render_impl(ctx, fg, bg, rays_d, image_indices_d, N, sphere_center3_d, sphere_radius3_d, include_xyz_real, cluster_2d,
                       z_steps_d, z_steps_bg_d, coarse_samples, u_fine_d, u_fine_bg_d, fine_samples, use_cascade, sh_deg, precision,
                       *out, workspace_d, workspace_bytes, stream, "mn_render_rays_bg_occ", occ, counts_out_d);
}

// Size queries: 0 for arguments the call would refuse.
size_t mn_render_rays_train_tape_bytes(const mn_model* m, int64_t N, int coarse_samples, int fine_samples, int use_cascade,
                                       int sh_deg, int precision) {
    if (!m || check_train(nullptr, m, N, coarse_samples, fine_samples, precision, "")) return 0;
    return make_train_plan(m, N, coarse_samples, fine_samples, use_cascade, sh_deg >= 0, precision == MN_PREC_TC_F16).tape_total;
}

size_t mn_render_rays_train_workspace_bytes(const mn_model* m, int64_t N, int coarse_samples, int fine_samples, int use_cascade,
                                            int sh_deg, int precision) {
    if (!m || check_train(nullptr, m, N, coarse_samples, fine_samples, precision, "")) return 0;
    return make_train_plan(m, N, coarse_samples, fine_samples, use_cascade, sh_deg >= 0, precision == MN_PREC_TC_F16).ws_total;
}

size_t mn_render_rays_train_backward_workspace_bytes(const mn_model* m, int64_t N, int coarse_samples, int fine_samples,
                                                     int use_cascade, int sh_deg, int precision) {
    if (!m || check_train(nullptr, m, N, coarse_samples, fine_samples, precision, "")) return 0;
    return make_train_plan(m, N, coarse_samples, fine_samples, use_cascade, sh_deg >= 0, precision == MN_PREC_TC_F16).bwd_total;
}

int mn_render_rays_train(mn_ctx* ctx, mn_model* m, const float* rays_d, const float* image_indices_d, int64_t N,
                         const float* z_steps_d, const float* jitter_d, float perturb, int coarse_samples,
                         const float* sigma_noise_coarse_d, const float* u_fine_d, const float* sigma_noise_fine_d, int fine_samples,
                         int use_cascade, int sh_deg, int precision, float* rgb_out_d, float* depth_out_d, float* depth_var_out_d,
                         float* rgb_coarse_out_d, void* tape_d, size_t tape_bytes, void* workspace_d, size_t workspace_bytes,
                         void* stream) {
    return train_impl(ctx, m, rays_d, image_indices_d, N, z_steps_d, jitter_d, perturb, coarse_samples, sigma_noise_coarse_d, u_fine_d,
                      sigma_noise_fine_d, fine_samples, use_cascade, sh_deg, precision, rgb_out_d, depth_out_d, depth_var_out_d,
                      rgb_coarse_out_d, tape_d, tape_bytes, workspace_d, workspace_bytes, (cudaStream_t)stream, "mn_render_rays_train");
}

int mn_render_rays_train_backward(mn_ctx* ctx, mn_model* m, int64_t N, int coarse_samples, int fine_samples, int use_cascade,
                                  int sh_deg, int precision, const float* grad_rgb_d, const float* grad_rgb_coarse_d,
                                  const void* tape_d, size_t tape_bytes, float* param_grads_d, void* workspace_d,
                                  size_t workspace_bytes, void* stream) {
    return train_backward_impl(ctx, m, N, coarse_samples, fine_samples, use_cascade, sh_deg, precision, grad_rgb_d, grad_rgb_coarse_d,
                               tape_d, tape_bytes, param_grads_d, workspace_d, workspace_bytes, (cudaStream_t)stream,
                               "mn_render_rays_train_backward");
}

size_t mn_render_rays_train_bg_tape_bytes(const mn_model* fg, const mn_model* bg, int64_t N, int coarse_samples, int fine_samples,
                                          int use_cascade, int sh_deg, int precision, int bg_precision) {
    if (!fg || !bg || check_train_bg(nullptr, fg, bg, N, coarse_samples, fine_samples, precision, bg_precision, "")) return 0;
    return make_bg_train_plan(fg, bg, N, coarse_samples, fine_samples, use_cascade, sh_deg >= 0, precision == MN_PREC_TC_F16,
                              bg_precision == MN_PREC_TC_F16).tape_total;
}

size_t mn_render_rays_train_bg_workspace_bytes(const mn_model* fg, const mn_model* bg, int64_t N, int coarse_samples, int fine_samples,
                                               int use_cascade, int sh_deg, int precision, int bg_precision) {
    if (!fg || !bg || check_train_bg(nullptr, fg, bg, N, coarse_samples, fine_samples, precision, bg_precision, "")) return 0;
    return make_bg_train_plan(fg, bg, N, coarse_samples, fine_samples, use_cascade, sh_deg >= 0, precision == MN_PREC_TC_F16,
                              bg_precision == MN_PREC_TC_F16).ws_total;
}

size_t mn_render_rays_train_bg_backward_workspace_bytes(const mn_model* fg, const mn_model* bg, int64_t N, int coarse_samples,
                                                        int fine_samples, int use_cascade, int sh_deg, int precision, int bg_precision) {
    if (!fg || !bg || check_train_bg(nullptr, fg, bg, N, coarse_samples, fine_samples, precision, bg_precision, "")) return 0;
    return make_bg_train_plan(fg, bg, N, coarse_samples, fine_samples, use_cascade, sh_deg >= 0, precision == MN_PREC_TC_F16,
                              bg_precision == MN_PREC_TC_F16).bwd_total;
}

int mn_render_rays_train_bg(mn_ctx* ctx, mn_model* fg, mn_model* bg, const float* rays_d, const float* image_indices_d, int64_t N,
                            const float* sphere_center3_d, const float* sphere_radius3_d, int include_xyz_real, int cluster_2d,
                            const float* z_steps_d, const float* z_steps_bg_d, const float* jitter_d, const float* jitter_bg_d,
                            float perturb, int coarse_samples, const float* sigma_noise_coarse_d, const float* sigma_noise_coarse_bg_d,
                            const float* u_fine_d, const float* u_fine_bg_d, const float* sigma_noise_fine_d,
                            const float* sigma_noise_fine_bg_d, int fine_samples, int use_cascade, int sh_deg, int precision,
                            int bg_precision, int bg_draws_by_ray, const mn_render_outputs* out, void* tape_d, size_t tape_bytes,
                            void* workspace_d, size_t workspace_bytes, void* stream) {
    return train_bg_impl(ctx, fg, bg, rays_d, image_indices_d, N, sphere_center3_d, sphere_radius3_d, include_xyz_real, cluster_2d,
                         z_steps_d, z_steps_bg_d, jitter_d, jitter_bg_d, perturb, coarse_samples, sigma_noise_coarse_d,
                         sigma_noise_coarse_bg_d, u_fine_d, u_fine_bg_d, sigma_noise_fine_d, sigma_noise_fine_bg_d, fine_samples,
                         use_cascade, sh_deg, precision, bg_precision, bg_draws_by_ray, out, tape_d, tape_bytes, workspace_d,
                         workspace_bytes, (cudaStream_t)stream, "mn_render_rays_train_bg");
}

int mn_render_rays_train_bg_backward(mn_ctx* ctx, mn_model* fg, mn_model* bg, int64_t N, int coarse_samples, int fine_samples,
                                     int use_cascade, int sh_deg, int precision, int bg_precision, const float* grad_rgb_d,
                                     const float* grad_rgb_coarse_d, const void* tape_d, size_t tape_bytes, float* param_grads_d,
                                     float* bg_param_grads_d, void* workspace_d, size_t workspace_bytes, void* stream) {
    return train_bg_backward_impl(ctx, fg, bg, N, coarse_samples, fine_samples, use_cascade, sh_deg, precision, bg_precision, grad_rgb_d,
                                  grad_rgb_coarse_d, tape_d, tape_bytes, param_grads_d, bg_param_grads_d, workspace_d, workspace_bytes,
                                  (cudaStream_t)stream, "mn_render_rays_train_bg_backward");
}

// ---- the training renders through an occupancy grid
size_t mn_render_rays_train_occ_tape_bytes(const mn_model* m, int64_t N, int coarse_samples, int fine_samples, int use_cascade,
                                           int sh_deg, int precision) {
    if (!m || check_train(nullptr, m, N, coarse_samples, fine_samples, precision, "")) return 0;
    return make_train_plan(m, N, coarse_samples, fine_samples, use_cascade, sh_deg >= 0, precision == MN_PREC_TC_F16, true).tape_total;
}

size_t mn_render_rays_train_occ_workspace_bytes(const mn_model* m, int64_t N, int coarse_samples, int fine_samples, int use_cascade,
                                                int sh_deg, int precision) {
    if (!m || check_train(nullptr, m, N, coarse_samples, fine_samples, precision, "")) return 0;
    return make_train_plan(m, N, coarse_samples, fine_samples, use_cascade, sh_deg >= 0, precision == MN_PREC_TC_F16, true).ws_total;
}

size_t mn_render_rays_train_occ_backward_workspace_bytes(const mn_model* m, int64_t N, int coarse_samples, int fine_samples,
                                                         int use_cascade, int sh_deg, int precision) {
    if (!m || check_train(nullptr, m, N, coarse_samples, fine_samples, precision, "")) return 0;
    return make_train_plan(m, N, coarse_samples, fine_samples, use_cascade, sh_deg >= 0, precision == MN_PREC_TC_F16, true).bwd_total;
}

int mn_render_rays_train_occ(mn_ctx* ctx, mn_model* m, const float* rays_d, const float* image_indices_d, int64_t N,
                             const float* z_steps_d, const float* jitter_d, float perturb, int coarse_samples,
                             const float* sigma_noise_coarse_d, const float* u_fine_d, const float* sigma_noise_fine_d, int fine_samples,
                             int use_cascade, int sh_deg, int precision, const mn_occupancy* occ, int32_t* counts_out_d, float* rgb_out_d,
                             float* depth_out_d, float* depth_var_out_d, float* rgb_coarse_out_d, void* tape_d, size_t tape_bytes,
                             void* workspace_d, size_t workspace_bytes, void* stream) {
    if (!occ) return mn_fail(ctx, MN_ERR_INVALID, "mn_render_rays_train_occ: occ is NULL");
    return train_impl(ctx, m, rays_d, image_indices_d, N, z_steps_d, jitter_d, perturb, coarse_samples, sigma_noise_coarse_d, u_fine_d,
                      sigma_noise_fine_d, fine_samples, use_cascade, sh_deg, precision, rgb_out_d, depth_out_d, depth_var_out_d,
                      rgb_coarse_out_d, tape_d, tape_bytes, workspace_d, workspace_bytes, (cudaStream_t)stream, "mn_render_rays_train_occ",
                      occ, counts_out_d);
}

int mn_render_rays_train_occ_backward(mn_ctx* ctx, mn_model* m, int64_t N, int coarse_samples, int fine_samples, int use_cascade,
                                      int sh_deg, int precision, const float* grad_rgb_d, const float* grad_rgb_coarse_d,
                                      const void* tape_d, size_t tape_bytes, float* param_grads_d, void* workspace_d,
                                      size_t workspace_bytes, void* stream) {
    return train_backward_impl(ctx, m, N, coarse_samples, fine_samples, use_cascade, sh_deg, precision, grad_rgb_d, grad_rgb_coarse_d,
                               tape_d, tape_bytes, param_grads_d, workspace_d, workspace_bytes, (cudaStream_t)stream,
                               "mn_render_rays_train_occ_backward", true);
}

size_t mn_render_rays_train_bg_occ_tape_bytes(const mn_model* fg, const mn_model* bg, int64_t N, int coarse_samples, int fine_samples,
                                              int use_cascade, int sh_deg, int precision, int bg_precision) {
    if (!fg || !bg || check_train_bg(nullptr, fg, bg, N, coarse_samples, fine_samples, precision, bg_precision, "")) return 0;
    return make_bg_train_plan(fg, bg, N, coarse_samples, fine_samples, use_cascade, sh_deg >= 0, precision == MN_PREC_TC_F16,
                              bg_precision == MN_PREC_TC_F16, true).tape_total;
}

size_t mn_render_rays_train_bg_occ_workspace_bytes(const mn_model* fg, const mn_model* bg, int64_t N, int coarse_samples,
                                                   int fine_samples, int use_cascade, int sh_deg, int precision, int bg_precision) {
    if (!fg || !bg || check_train_bg(nullptr, fg, bg, N, coarse_samples, fine_samples, precision, bg_precision, "")) return 0;
    return make_bg_train_plan(fg, bg, N, coarse_samples, fine_samples, use_cascade, sh_deg >= 0, precision == MN_PREC_TC_F16,
                              bg_precision == MN_PREC_TC_F16, true).ws_total;
}

size_t mn_render_rays_train_bg_occ_backward_workspace_bytes(const mn_model* fg, const mn_model* bg, int64_t N, int coarse_samples,
                                                            int fine_samples, int use_cascade, int sh_deg, int precision,
                                                            int bg_precision) {
    if (!fg || !bg || check_train_bg(nullptr, fg, bg, N, coarse_samples, fine_samples, precision, bg_precision, "")) return 0;
    return make_bg_train_plan(fg, bg, N, coarse_samples, fine_samples, use_cascade, sh_deg >= 0, precision == MN_PREC_TC_F16,
                              bg_precision == MN_PREC_TC_F16, true).bwd_total;
}

int mn_render_rays_train_bg_occ(mn_ctx* ctx, mn_model* fg, mn_model* bg, const float* rays_d, const float* image_indices_d, int64_t N,
                                const float* sphere_center3_d, const float* sphere_radius3_d, int include_xyz_real, int cluster_2d,
                                const float* z_steps_d, const float* z_steps_bg_d, const float* jitter_d, const float* jitter_bg_d,
                                float perturb, int coarse_samples, const float* sigma_noise_coarse_d,
                                const float* sigma_noise_coarse_bg_d, const float* u_fine_d, const float* u_fine_bg_d,
                                const float* sigma_noise_fine_d, const float* sigma_noise_fine_bg_d, int fine_samples, int use_cascade,
                                int sh_deg, int precision, int bg_precision, const mn_occupancy* occ, int32_t* counts_out_d,
                                int bg_draws_by_ray, const mn_render_outputs* out, void* tape_d, size_t tape_bytes, void* workspace_d,
                                size_t workspace_bytes, void* stream) {
    if (!occ) return mn_fail(ctx, MN_ERR_INVALID, "mn_render_rays_train_bg_occ: occ is NULL");
    return train_bg_impl(ctx, fg, bg, rays_d, image_indices_d, N, sphere_center3_d, sphere_radius3_d, include_xyz_real, cluster_2d,
                         z_steps_d, z_steps_bg_d, jitter_d, jitter_bg_d, perturb, coarse_samples, sigma_noise_coarse_d,
                         sigma_noise_coarse_bg_d, u_fine_d, u_fine_bg_d, sigma_noise_fine_d, sigma_noise_fine_bg_d, fine_samples,
                         use_cascade, sh_deg, precision, bg_precision, bg_draws_by_ray, out, tape_d, tape_bytes, workspace_d,
                         workspace_bytes, (cudaStream_t)stream, "mn_render_rays_train_bg_occ", occ, counts_out_d);
}

int mn_render_rays_train_bg_occ_backward(mn_ctx* ctx, mn_model* fg, mn_model* bg, int64_t N, int coarse_samples, int fine_samples,
                                         int use_cascade, int sh_deg, int precision, int bg_precision, const float* grad_rgb_d,
                                         const float* grad_rgb_coarse_d, const void* tape_d, size_t tape_bytes, float* param_grads_d,
                                         float* bg_param_grads_d, void* workspace_d, size_t workspace_bytes, void* stream) {
    return train_bg_backward_impl(ctx, fg, bg, N, coarse_samples, fine_samples, use_cascade, sh_deg, precision, bg_precision, grad_rgb_d,
                                  grad_rgb_coarse_d, tape_d, tape_bytes, param_grads_d, bg_param_grads_d, workspace_d, workspace_bytes,
                                  (cudaStream_t)stream, "mn_render_rays_train_bg_occ_backward", true);
}

// bits = pack(sigmas >= thresh): one warp per 32 cells, each lane's comparison balloted into the cells' word.  A NaN sigma fails
// the comparison (an empty cell), as torch's does.
int mn_occupancy_pack(mn_ctx* ctx, const float* sigmas_d, int64_t n, float thresh, uint32_t* bits_d, void* stream) {
    if (!ctx || n < 0 || (n > 0 && (!sigmas_d || !bits_d))) return MN_ERR_INVALID;
    if (n == 0) return MN_OK;
    occ_pack_kernel<<<(unsigned)mn_cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(sigmas_d, n, thresh, bits_d);
    MN_LAUNCH_CHECK(ctx);
    return MN_OK;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------
// Fused per-ray all-gather (SURVEY.md §8e, "fused form"): every rank stores its rays' (rgb, depth) rows straight into
// EVERY rank's result buffer through peer-mapped pointers (NVLink / NVSwitch P2P stores), instead of packing them and
// calling a collective.  The buffers are symmetric allocations exchanged by the host (torch symmetric memory in the
// Python mirror); ordering between ranks is the caller's barrier pair (see mega_nerf_b200/dist.py::PeerGather).
// ------------------------------------------------------------------------------------------------
#define MN_MAX_PEERS 16
struct PeerBufs {
    float* p[MN_MAX_PEERS];
};

__global__ void peer_gather_store_kernel(const float* __restrict__ rgb, const float* __restrict__ depth, int64_t n, int64_t row0,
                                         PeerBufs bufs, int G) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 v = make_float4(rgb[i * 3 + 0], rgb[i * 3 + 1], rgb[i * 3 + 2], depth ? depth[i] : 0.0f);
    for (int g = 0; g < G; ++g) reinterpret_cast<float4*>(bufs.p[g])[row0 + i] = v;   // 16-byte store per peer
}

extern "C" int mn_peer_gather_store(mn_ctx* ctx, const float* rgb_d, const float* depth_d, int64_t n, int64_t row0,
                                    const void* const* peer_bufs, int n_peers, void* stream) {
    if (!ctx || !rgb_d || !peer_bufs || n < 0 || row0 < 0 || n_peers < 1 || n_peers > MN_MAX_PEERS) return MN_ERR_INVALID;
    if (n == 0) return MN_OK;
    PeerBufs b{};
    for (int g = 0; g < n_peers; ++g) {
        if (!peer_bufs[g]) return mn_fail(ctx, MN_ERR_INVALID, "mn_peer_gather_store: null peer buffer");
        b.p[g] = (float*)peer_bufs[g];
    }
    peer_gather_store_kernel<<<(unsigned)mn_cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(rgb_d, depth_d, n, row0, b, n_peers);
    MN_LAUNCH_CHECK(ctx);
    return MN_OK;
}
