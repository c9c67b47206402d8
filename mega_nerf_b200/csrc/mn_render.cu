// mn_render_rays / mn_render_rays_bg: the inference path of render_rays (rendering.py:15-248, eval mode) as ONE C call - coarse
// depths -> model query -> weights -> inverse-CDF resampling -> fine query -> merge + volume rendering, and with a background
// (NeRF++) network its pass too (rendering.py:34-62, 143-173): sphere split, inverted-sphere points, flipped two-pass render and
// the lambda blend.  It only sequences the stage kernels of this library on the caller's stream, from a caller-provided
// workspace: no allocation, no host sync, ~20 (foreground) / ~40 (with background) launches issued back to back without
// returning to the host language in between (the Python mirror spends 1.6-2.0 ms of interpreter time on the foreground alone).
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

constexpr int kSplitBlock = 1024;

// Background split, per ray (render.py `_render`, rendering.py:34-47): fg_far = max(sphere exit, near); the ray reaches the
// background iff far > fg_far; its last delta (fg_far, else 1e10) and the foreground far override min(far, fg_far).  flag[i] = 1
// for a background ray (turned into its compacted position by bg_compact_kernel); blk[b] = background rays of block b.
__global__ void __launch_bounds__(kSplitBlock) bg_split_kernel(const float* __restrict__ rays, const float* __restrict__ center,
                                                               const float* __restrict__ radius, int64_t N, float* __restrict__ far_ov,
                                                               float* __restrict__ last_delta, int* __restrict__ flag,
                                                               int* __restrict__ blk, unsigned int* status) {
    const int64_t i = (int64_t)blockIdx.x * kSplitBlock + threadIdx.x;
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
__global__ void __launch_bounds__(kSplitBlock) bg_compact_kernel(const float* __restrict__ rays, const float* __restrict__ idx,
                                                                 int64_t N, const int* __restrict__ blk, int* __restrict__ pos,
                                                                 int64_t* __restrict__ ids, float* __restrict__ dirs,
                                                                 float* __restrict__ cidx, int* __restrict__ count) {
    __shared__ int wsum[32], wbase[32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int part = 0;                                           // background rays of the blocks before this one
    for (unsigned b = threadIdx.x; b < blockIdx.x; b += kSplitBlock) part += blk[b];
    for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
    const int64_t i = (int64_t)blockIdx.x * kSplitBlock + threadIdx.x;
    const bool with_bg = i < N && pos[i] != 0;
    const unsigned bal = __ballot_sync(0xffffffffu, with_bg);
    if (lane == 0) { wsum[warp] = part; wbase[warp] = __popc(bal); }
    __syncthreads();
    if (threadIdx.x == 0) {
        int run = 0;
        for (int w = 0; w < kSplitBlock / 32; ++w) run += wsum[w];
        for (int w = 0; w < kSplitBlock / 32; ++w) { const int c = wbase[w]; wbase[w] = run; run += c; }
        if (blockIdx.x == gridDim.x - 1) *count = run;
    }
    __syncthreads();
    if (i >= N) return;
    int p = -1;
    if (with_bg) {
        p = wbase[warp] + __popc(bal & ((1u << lane) - 1));
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

struct RenderPlan {
    int64_t N;
    int Sc, Sf, Sq;            // coarse samples, fine draws, samples of the fine query (Sf, or Sc + Sf under cascade)
    int out_cols;              // columns of the raw model output (rgb_dim + 1)
    size_t z_c, xyz_c, mlp_c, raw_c, w_c, z_f, z_q, xyz_f, mlp_f, raw_f, last_delta, model_ws, total;
    size_t model_ws_bytes;
    // background pass: Sb coarse samples (Sc / 2), Fb fine draws (Sf / 2), Sqb samples of its fine query; every per-ray buffer
    // holds N rays (the compacted background rays first)
    int Sb, Fb, Sqb;
    size_t far_ov, pos, blk, count, ids, dirs, idx, zb, zb_flip, xyz_b, dreal_b, mlp_b, raw_b, w_b, zf_b, zq_b, zq_b_flip, xyz_fb,
        dreal_fb, mlp_fb, raw_fb, ld_b, rgb_b, depth_b, rgb_cb, lam, lam_c;
};

RenderPlan make_plan(const mn_model* m, const mn_model* bg, int64_t N, int Sc, int Sf, int use_cascade, int sh, int precision) {
    RenderPlan p{};
    p.N = N; p.Sc = Sc; p.Sf = Sf;
    p.Sq = Sf > 0 ? (use_cascade ? Sc + Sf : Sf) : 0;
    p.out_cols = m->nd.rgb_dim + 1;
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off += mn_align(bytes); return o; };
    p.z_c = take((size_t)N * Sc * 4);
    p.xyz_c = take((size_t)N * Sc * 12);
    p.mlp_c = sh ? take((size_t)N * Sc * p.out_cols * 4) : 0;      // raw SH coefficients before the head
    p.raw_c = take((size_t)N * Sc * 16);
    p.w_c = take((size_t)N * Sc * 4);
    p.z_f = take((size_t)N * (Sf > 0 ? Sf : 1) * 4);
    p.z_q = use_cascade && Sf > 0 ? take((size_t)N * p.Sq * 4) : p.z_f;
    p.xyz_f = take((size_t)N * (p.Sq > 0 ? p.Sq : 1) * 12);
    p.mlp_f = sh ? take((size_t)N * (p.Sq > 0 ? p.Sq : 1) * p.out_cols * 4) : 0;
    p.raw_f = take((size_t)N * (p.Sq > 0 ? p.Sq : 1) * 16);
    p.last_delta = take((size_t)N * 4);
    const size_t a = mn_model_workspace_bytes(m, N * Sc, precision);
    const size_t b = p.Sq > 0 ? mn_model_workspace_bytes(m, N * p.Sq, precision) : 0;
    p.model_ws_bytes = a > b ? a : b;
    if (bg) {
        p.Sb = Sc / 2;
        p.Fb = Sf / 2;
        p.Sqb = p.Fb > 0 ? (use_cascade ? p.Sb + p.Fb : p.Fb) : 0;
        const int Sb = p.Sb > 0 ? p.Sb : 1, Sqb = p.Sqb > 0 ? p.Sqb : 1, bcols = bg->nd.rgb_dim + 1;
        p.far_ov = take((size_t)N * 4);
        p.pos = take((size_t)N * 4);
        p.blk = take((size_t)mn_cdiv(N, kSplitBlock) * 4);
        p.count = take(4);
        p.ids = take((size_t)N * 8);
        p.dirs = take((size_t)N * 12);
        p.idx = take((size_t)N * 4);
        p.zb = take((size_t)N * Sb * 4);
        p.zb_flip = take((size_t)N * Sb * 4);
        p.xyz_b = take((size_t)N * Sb * 28);                            // 7 columns with the real-xyz prefix, else 4
        p.dreal_b = take((size_t)N * Sb * 4);
        p.mlp_b = sh ? take((size_t)N * Sb * bcols * 4) : 0;
        p.raw_b = take((size_t)N * Sb * 16);
        p.w_b = take((size_t)N * Sb * 4);
        p.zf_b = take((size_t)N * (p.Fb > 0 ? p.Fb : 1) * 4);
        p.zq_b = use_cascade && p.Fb > 0 ? take((size_t)N * Sqb * 4) : p.zf_b;
        p.zq_b_flip = use_cascade && p.Fb > 0 ? take((size_t)N * Sqb * 4) : 0;
        p.xyz_fb = take((size_t)N * Sqb * 28);
        p.dreal_fb = take((size_t)N * Sqb * 4);
        p.mlp_fb = sh ? take((size_t)N * Sqb * bcols * 4) : 0;
        p.raw_fb = take((size_t)N * Sqb * 16);
        p.ld_b = take((size_t)N * 4);
        p.rgb_b = take((size_t)N * 12);
        p.depth_b = take((size_t)N * 4);
        p.rgb_cb = take((size_t)N * 12);
        p.lam = take((size_t)N * 4);
        p.lam_c = take((size_t)N * 4);
        const size_t c = mn_model_workspace_bytes(bg, N * Sb, precision);
        const size_t d = p.Sqb > 0 ? mn_model_workspace_bytes(bg, N * p.Sqb, precision) : 0;
        if (c > p.model_ws_bytes) p.model_ws_bytes = c;
        if (d > p.model_ws_bytes) p.model_ws_bytes = d;
    }
    p.model_ws = take(p.model_ws_bytes);
    p.total = off + 256;
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

int render_impl(mn_ctx* ctx, mn_model* m, mn_model* bg, const float* rays_d, const float* image_indices_d, int64_t N,
                const float* center_d, const float* radius_d, int include_xyz_real, int cluster_2d, const float* z_steps_d,
                const float* z_steps_bg_d, int coarse_samples, const float* u_fine_d, const float* u_fine_bg_d, int fine_samples,
                int use_cascade, int sh_deg, int precision, const mn_render_outputs& o, void* workspace_d, size_t workspace_bytes,
                void* stream, const char* name) {
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
    if (N == 0) return MN_OK;
    const bool sh = sh_deg >= 0;
    const RenderPlan p = make_plan(m, bg, N, coarse_samples, fine_samples, use_cascade, sh, precision);
    if (!workspace_d || workspace_bytes < p.total) return mn_fail(ctx, MN_ERR_WORKSPACE, nm + ": workspace too small");
    char* W = (char*)workspace_d;
    auto F = [&](size_t off) { return reinterpret_cast<float*>(W + off); };
    auto I = [&](size_t off) { return reinterpret_cast<int*>(W + off); };
    cudaStream_t st = (cudaStream_t)stream;
    const int Sc = p.Sc, Sf = p.Sf, Sq = p.Sq;
    const bool fine = Sf > 0;
    const bool want_depth = o.depth || o.depth_var;
    float* rgb_out_d = o.rgb;
    float* depth_out_d = o.depth;
    float* depth_var_out_d = o.depth_var;
    float* rgb_coarse_out_d = o.rgb_coarse;

    // one model query on [n, S, cols] points -> raw [n, S, 4]   (rendering.py:275-334).  dirs / idx: per ray; live: the rays
    // that hold data (background pass) or all n.
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
        int r = live ? mn_model_forward_live(ctx, net, &rows, N * S, lr, coarse, precision, out, W + p.model_ws, p.model_ws_bytes, st)
                     : mn_model_forward(ctx, net, &rows, N * S, coarse, 0, nullptr, precision, out, W + p.model_ws, p.model_ws_bytes, stream);
        if (r) return r;
        if (sh) return mn_stage_sh_to_rgb(ctx, sh_deg, mlp_out, net->nd.rgb_dim + 1, dirs, dstride, S, N * S, 1, lr, raw_out, st);
        return MN_OK;
    };

    if (!bg) {
        fill_kernel<<<(unsigned)mn_cdiv(N, 256), 256, 0, st>>>(F(p.last_delta), N, 1e10f);   // no background: rendering.py:33
        MN_LAUNCH_CHECK(ctx);
    } else {
        // ---- split and compaction (render.py:292-299)
        const unsigned nblk = (unsigned)mn_cdiv(N, kSplitBlock);
        bg_split_kernel<<<nblk, kSplitBlock, 0, st>>>(rays_d, center_d, radius_d, N, F(p.far_ov), F(p.last_delta), I(p.pos), I(p.blk),
                                                     ctx->status_d);
        MN_LAUNCH_CHECK(ctx);
        float* bidx = image_indices_d ? F(p.idx) : nullptr;
        bg_compact_kernel<<<nblk, kSplitBlock, 0, st>>>(rays_d, image_indices_d, N, I(p.blk), I(p.pos),
                                                       reinterpret_cast<int64_t*>(W + p.ids), F(p.dirs), bidx, I(p.count));
        MN_LAUNCH_CHECK(ctx);
        fill_kernel<<<(unsigned)mn_cdiv(N, 256), 256, 0, st>>>(F(p.ld_b), N, 1e10f);            // no bg_lambda in this pass
        MN_LAUNCH_CHECK(ctx);

        // ---- background pass over the compacted rays (render.py:300-312 -> _two_pass with flip):  coarse depths from
        // z_steps_bg; query and composite see them flipped, with the unflipped real depths (quirk of the reference)
        const int* cnt = I(p.count);
        const LiveRows lr{cnt, 1};
        const int64_t* ids = reinterpret_cast<const int64_t*>(W + p.ids);
        const int Sb = p.Sb, Fb = p.Fb, Sqb = p.Sqb, cols = include_xyz_real ? 7 : 4;
        const bool bfine = Fb > 0;
        if ((rc = mn_stage_stratify(ctx, z_steps_bg_d, 0, nullptr, 0.0f, N, Sb, 0, lr, F(p.zb), st))) return rc;
        if ((rc = mn_stage_stratify(ctx, z_steps_bg_d, 0, nullptr, 0.0f, N, Sb, 1, lr, F(p.zb_flip), st))) return rc;
        if ((rc = mn_stage_points_outside(ctx, rays_d, ids, F(p.zb), center_d, radius_d, N, Sb, include_xyz_real, cluster_2d, 1, lr,
                                          F(p.xyz_b), F(p.dreal_b), st)))
            return rc;
        if ((rc = query(bg, F(p.xyz_b), cols, Sb, 1, F(p.mlp_b), F(p.raw_b), F(p.dirs), 3, bidx, cnt))) return rc;
        if ((rc = mn_stage_composite(ctx, F(p.raw_b), F(p.zb_flip), F(p.dreal_b), Sb, nullptr, nullptr, nullptr, 0, F(p.ld_b), N, 1, lr,
                                     bfine ? F(p.w_b) : nullptr, use_cascade ? (bfine ? F(p.rgb_cb) : F(p.rgb_b)) : nullptr,
                                     (!bfine && depth_out_d) ? F(p.depth_b) : nullptr, nullptr, nullptr, st)))
            return rc;
        if (bfine) {
            // resampling from the unflipped bins with the weights in flipped order (quirk Q7), then points outside the sphere
            if ((rc = mn_stage_sample_pdf(ctx, F(p.zb), F(p.w_b), Sb, nullptr, u_fine_bg_d, 0, N, Sb, Fb, lr, F(p.zf_b), nullptr, nullptr, st))) return rc;
            if (use_cascade)
                if ((rc = mn_stage_sort_cat(ctx, F(p.zb), Sb, F(p.zf_b), Fb, N, 0, lr, F(p.zq_b), F(p.zq_b_flip), st))) return rc;
            if ((rc = mn_stage_points_outside(ctx, rays_d, ids, F(p.zq_b), center_d, radius_d, N, Sqb, include_xyz_real, cluster_2d,
                                              use_cascade ? 1 : 0, lr, F(p.xyz_fb), F(p.dreal_fb), st)))
                return rc;
            if ((rc = query(bg, F(p.xyz_fb), cols, Sqb, 0, F(p.mlp_fb), F(p.raw_fb), F(p.dirs), 3, bidx, cnt))) return rc;
            float* bdepth = depth_out_d ? F(p.depth_b) : nullptr;
            if (use_cascade)
                rc = mn_stage_composite(ctx, F(p.raw_fb), F(p.zq_b_flip), F(p.dreal_fb), Sqb, nullptr, nullptr, nullptr, 0, F(p.ld_b), N,
                                        1, lr, nullptr, F(p.rgb_b), bdepth, nullptr, nullptr, st);
            else
                rc = mn_stage_composite(ctx, F(p.raw_fb), F(p.zf_b), F(p.dreal_fb), Fb, F(p.raw_b), F(p.zb_flip), F(p.dreal_b), Sb,
                                        F(p.ld_b), N, 1, lr, nullptr, F(p.rgb_b), bdepth, nullptr, nullptr, st);
            if (rc) return rc;
        }
    }
    const float* far_ov = bg ? F(p.far_ov) : nullptr;
    // bg_lambda of the final type and of the cascade's coarse type (render.py:317: requested iff there is a background)
    float* lam = bg ? (o.bg_lambda ? o.bg_lambda : F(p.lam)) : nullptr;
    float* lam_c = (bg && use_cascade && fine) ? (o.bg_lambda_coarse ? o.bg_lambda_coarse : F(p.lam_c)) : nullptr;

    // ---- coarse pass (rendering.py:82-87, 190-205)
    if ((rc = mn_sample_coarse(ctx, rays_d, far_ov, z_steps_d, nullptr, 0.0f, N, Sc, F(p.z_c), F(p.xyz_c), stream))) return rc;
    if ((rc = query(m, F(p.xyz_c), 3, Sc, 1, F(p.mlp_c), F(p.raw_c), rays_d + 3, 8, image_indices_d, nullptr))) return rc;
    if ((rc = mn_composite(ctx, F(p.raw_c), F(p.z_c), nullptr, Sc, nullptr, nullptr, nullptr, 0, F(p.last_delta), N, 0,
                           fine ? F(p.w_c) : nullptr, use_cascade ? (fine ? rgb_coarse_out_d : rgb_out_d) : nullptr,
                           (!fine && want_depth) ? (depth_out_d ? depth_out_d : F(p.w_c)) : nullptr,
                           !fine ? depth_var_out_d : nullptr, use_cascade ? (fine ? lam_c : lam) : nullptr, stream)))
        return rc;

    if (fine) {
        // ---- resample (rendering.py:207-223) and fine pass (:224-243)
        if ((rc = mn_sample_pdf(ctx, F(p.z_c), F(p.w_c), Sc, nullptr, u_fine_d, 0, N, Sc, Sf, F(p.z_f), nullptr, nullptr, stream))) return rc;
        if (use_cascade)
            if ((rc = mn_sort_cat(ctx, F(p.z_c), Sc, F(p.z_f), Sf, N, 0, F(p.z_q), stream))) return rc;
        if ((rc = mn_points_from_z(ctx, rays_d, F(p.z_q), N, Sq, F(p.xyz_f), stream))) return rc;
        if ((rc = query(m, F(p.xyz_f), 3, Sq, 0, F(p.mlp_f), F(p.raw_f), rays_d + 3, 8, image_indices_d, nullptr))) return rc;
        // depth scratch when only the variance is wanted: the coarse weights are dead by now
        float* depth_dst = want_depth ? (depth_out_d ? depth_out_d : F(p.w_c)) : nullptr;
        if (use_cascade)
            rc = mn_composite(ctx, F(p.raw_f), F(p.z_q), nullptr, Sq, nullptr, nullptr, nullptr, 0, F(p.last_delta), N, 0, nullptr,
                              rgb_out_d, depth_dst, depth_var_out_d, lam, stream);
        else
            rc = mn_composite(ctx, F(p.raw_f), F(p.z_f), nullptr, Sf, F(p.raw_c), F(p.z_c), nullptr, Sc, F(p.last_delta), N, 0, nullptr,
                              rgb_out_d, depth_dst, depth_var_out_d, lam, stream);
        if (rc) return rc;
    }
    if (!bg) return MN_OK;

    // ---- blend (render.py:320-340): the final type's rgb / depth, and rgb_coarse under cascade with fine samples
    auto blend = [&](float* val, const float* bval, const float* l, int C, float* fg_out, float* bg_out) -> int {
        bg_blend_kernel<<<(unsigned)mn_cdiv(N * C, 256), 256, 0, st>>>(val, bval, l, I(p.pos), N, C, fg_out, bg_out);
        MN_LAUNCH_CHECK(ctx);
        return MN_OK;
    };
    if ((rc = blend(rgb_out_d, F(p.rgb_b), lam, 3, o.fg_rgb, o.bg_rgb))) return rc;
    if (depth_out_d)
        if ((rc = blend(depth_out_d, F(p.depth_b), lam, 1, o.fg_depth, o.bg_depth))) return rc;
    if (use_cascade && fine && rgb_coarse_out_d)
        if ((rc = blend(rgb_coarse_out_d, F(p.rgb_cb), lam_c, 3, o.fg_rgb_coarse, o.bg_rgb_coarse))) return rc;
    return MN_OK;
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
