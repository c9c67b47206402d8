// Context / model management and the nn.Module-level forward entry point of the C ABI.
#include <cuda_fp16.h>

#include <cstring>
#include <vector>

#include "mn_model.cuh"

namespace {

// Element i of one re-layout (PackOp).
__device__ __forceinline__ void pack_elem(const PackOp& op, long long i) {
    const float* __restrict__ src = op.src;
    switch (op.kind) {
        case PK_COPY:
            reinterpret_cast<float*>(op.dst)[i] = src[i];
            break;
        case PK_TRANSPOSE: {      // src [N][K] (nn.Linear weight, [out,in]) -> dst [K][N]
            const int N = op.p[0], K = op.p[1];
            const int k = (int)(i / N), n = (int)(i % N);
            reinterpret_cast<float*>(op.dst)[i] = src[(long long)n * K + k];
            break;
        }
        case PK_SUBMATRIX: {      // src [N][K] -> dst [N][kw] = src[:, koff : koff + kw]
            const int K = op.p[1], koff = op.p[2], kw = op.p[3];
            const int n = (int)(i / kw), k = (int)(i % kw);
            reinterpret_cast<float*>(op.dst)[i] = src[(long long)n * K + koff + k];
            break;
        }
        // K-major Wt[k][n_src] fp32 -> the tensor-core image [N/nw][K/8][nw][8] fp16, optional fp16 residual (lo).  Source
        // column ks of image column k: the first k_pad0 image columns hold k_real0 source columns and zero padding, the rest
        // follow contiguously; columns and rows past the source are zero.
        case PK_TC_HALF: {
            const int n_src = op.p[0], k_src = op.p[1], K = op.p[3], k_real0 = op.p[4], k_pad0 = op.p[5], nw = op.p[6];
            const int k8 = (int)(i % 8), n = (int)((i / 8) % nw);
            const long long rest = i / (8 * (long long)nw);
            const int kc = (int)(rest % (K / 8)), hh = (int)(rest / (K / 8));
            const int k = kc * 8 + k8, ng = hh * nw + n;
            int ks;
            if (k < k_pad0) ks = k < k_real0 ? k : -1;
            else ks = k_real0 + (k - k_pad0);
            float v = 0.0f;
            if (ks >= 0 && ks < k_src && ng < n_src) v = src[(long long)ks * n_src + ng];
            const __half h = __float2half_rn(v);
            reinterpret_cast<__half*>(op.dst)[i] = h;
            if (op.dst2) reinterpret_cast<__half*>(op.dst2)[i] = __float2half_rn(v - __half2float(h));
            break;
        }
        case PK_TC_F32:           // copy with zero padding
            reinterpret_cast<float*>(op.dst)[i] = i < op.p[0] ? src[i] : 0.0f;
            break;
        case PK_RGBW: {           // K-major Wt[k][c] -> [c][k], rows p[2] floats apart (0: K)
            const int K = op.p[0], Cc = op.p[1], ld = op.p[2] > 0 ? op.p[2] : K;
            reinterpret_cast<float*>(op.dst)[(i % Cc) * ld + i / Cc] = src[i];
            break;
        }
    }
}

__global__ void __launch_bounds__(256) pack_ops_kernel(const PackOp* __restrict__ ops) {
    const PackOp op = ops[blockIdx.y];
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < op.count; i += (long long)gridDim.x * blockDim.x)
        pack_elem(op, i);
}

// mn_model_repack: one launch over a resident table of every sub-module's re-layouts, cut into chunks of kRepackChunk elements
// so that the blocks share the work evenly whatever the sizes of the ops (a 2048 x 2048 weight and a 1-float bias alike).
// first[j] is the first chunk of op j (first[n_ops] = the launch's chunks); block b runs chunk b of the op that holds it.
constexpr int kRepackChunk = 4096;

__global__ void __launch_bounds__(256) repack_kernel(const PackOp* __restrict__ ops, const long long* __restrict__ first, int n_ops) {
    const long long b = blockIdx.x;
    int lo = 0, hi = n_ops - 1;              // the last op whose first chunk is <= b (ops of no chunk are skipped over)
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (first[mid] <= b) lo = mid;
        else hi = mid - 1;
    }
    const PackOp op = ops[lo];
    const long long i0 = (b - first[lo]) * kRepackChunk;
    const long long i1 = op.count < i0 + kRepackChunk ? op.count : i0 + kRepackChunk;
    for (long long i = i0 + threadIdx.x; i < i1; i += 256) pack_elem(op, i);
}

void pack_T(mn_ctx* ctx, const float* src, int N, int K, float* dst) {
    mn_pack_push(ctx, PackOp{src, dst, nullptr, (long long)N * K, PK_TRANSPOSE, {N, K, 0, 0, 0, 0, 0}});
}

void pack_sub(mn_ctx* ctx, const float* src, int N, int K, int koff, int kw, float* dst) {
    if ((long long)N * kw == 0) return;
    mn_pack_push(ctx, PackOp{src, dst, nullptr, (long long)N * kw, PK_SUBMATRIX, {N, K, koff, kw, 0, 0, 0}});
}

int al4(int x) { return (x + 3) / 4 * 4; }

void build_layout(mn_model* m) {
    const mn_model_desc& d = m->d;
    NetDims& nd = m->nd;
    nd.layers = d.layers;
    nd.L = d.layer_dim;
    nd.xyz_dim = d.xyz_dim;
    nd.nf_xyz = d.pos_xyz_dim;
    nd.nf_dir = d.pos_dir_dim;
    nd.in_xyz = d.xyz_dim + d.xyz_dim * d.pos_xyz_dim * 2;
    nd.in_dir = d.pos_dir_dim > 0 ? 3 + 3 * d.pos_dir_dim * 2 : 0;
    nd.app = d.appearance_dim;
    nd.affine = d.affine_appearance;
    nd.app_in_dira = (d.appearance_dim > 0 && !d.affine_appearance) ? 1 : 0;
    nd.aux = nd.in_dir + (nd.app_in_dira ? nd.app : 0);
    nd.has_dir_a = (d.pos_dir_dim > 0 || nd.app_in_dira) ? 1 : 0;
    nd.rgb_dim = d.rgb_dim;
    nd.rgb_in = nd.has_dir_a ? nd.L / 2 : nd.L;
    nd.softplus = d.shifted_softplus;
    nd.app_count = d.appearance_count;
    nd.skip_mask = 0;
    for (int i = 0; i < d.n_skip; ++i)
        if (d.skip_layers[i] > 0 && d.skip_layers[i] < 32) nd.skip_mask |= 1 << d.skip_layers[i];

    PackedLayout& l = m->lay;
    int off = 0;
    auto take = [&](int n) { int o = off; off += al4(n); return o; };
    for (int i = 0; i < nd.layers; ++i) {
        l.kin[i] = (i == 0) ? nd.in_xyz : (((nd.skip_mask >> i) & 1) ? nd.in_xyz + nd.L : nd.L);
        l.w[i] = take(l.kin[i] * nd.L);
        l.b[i] = take(nd.L);
    }
    l.sigma_w = take(nd.L);
    l.sigma_b = take(1);
    l.final_w = take(nd.has_dir_a ? nd.L * nd.L : 0);
    l.final_b = take(nd.has_dir_a ? nd.L : 0);
    l.dira_w = take(nd.has_dir_a ? (nd.L + nd.aux) * (nd.L / 2) : 0);
    l.dira_b = take(nd.has_dir_a ? nd.L / 2 : 0);
    l.rgb_w = take(nd.rgb_in * nd.rgb_dim);
    l.rgb_b = take(nd.rgb_dim);
    l.emb = take(nd.app > 0 ? nd.app_count * nd.app : 0);
    l.aff_w = take(nd.affine ? nd.app * 12 : 0);
    l.aff_b = take(nd.affine ? 12 : 0);
    l.total = off;

    // training tapes (mn_model.cuh)
    TapeLayout& t = m->tape;
    int c = 0;
    auto chan = [&](int n) { int o = c; c += n; return o; };
    t.a_pe = chan(nd.in_xyz);
    t.a_aux = chan(nd.aux);
    t.a_h = chan(nd.layers * nd.L);
    t.a_f = chan(nd.has_dir_a ? nd.L : 0);
    t.a_g = chan(nd.has_dir_a ? nd.L / 2 : 0);
    t.a_rgb = chan(nd.rgb_dim);
    t.a_lin = chan(nd.affine ? 3 : 0);
    t.a_sig = chan(1);
    t.a_id = chan(nd.app > 0 ? 1 : 0);
    t.a_total = c;
    c = 0;
    t.g_z = chan(nd.layers * nd.L);
    t.g_final = chan(nd.has_dir_a ? nd.L : 0);
    t.g_dira = chan(nd.has_dir_a ? nd.L / 2 : 0);
    t.g_rgb = chan(nd.rgb_dim);
    t.g_sig = chan(1);
    t.g_total = c;

    BwdLayout& bl = m->blay;
    off = 0;
    bl.w[0] = 0;
    for (int i = 1; i < nd.layers; ++i) bl.w[i] = take(nd.L * nd.L);
    bl.final_w = take(nd.has_dir_a ? nd.L * nd.L : 0);
    bl.dira_f = take(nd.has_dir_a ? (nd.L / 2) * nd.L : 0);
    bl.dira_e = take(nd.app_in_dira ? (nd.L / 2) * nd.app : 0);
    bl.total = off > 0 ? off : 4;
    m->tc = tc_net(*m);      // the tensor-core plan, from the layouts above
}

}  // namespace

void mn_pack_push(mn_ctx* ctx, const PackOp& op) { ctx->pack_ops.push_back(op); }

int mn_pack_flush(mn_ctx* ctx, cudaStream_t st) {
    const size_t n = ctx->pack_ops.size();
    if (n == 0) return MN_OK;
    if (n > ctx->pack_ops_cap) {
        if (ctx->pack_ops_d) {
            MN_CUDA(ctx, cudaStreamSynchronize(st));      // a previous table may still be read
            cudaFree(ctx->pack_ops_d);
        }
        ctx->pack_ops_cap = n < 128 ? 128 : 2 * n;
        MN_CUDA(ctx, cudaMalloc(&ctx->pack_ops_d, ctx->pack_ops_cap * 2 * sizeof(PackOp)));
    }
    // two alternating halves of the table: the launch of the previous flush may still be reading its half
    static thread_local unsigned flip = 0;
    PackOp* tab = ctx->pack_ops_d + (flip++ & 1u) * ctx->pack_ops_cap;
    MN_CUDA(ctx, cudaMemcpyAsync(tab, ctx->pack_ops.data(), n * sizeof(PackOp), cudaMemcpyHostToDevice, st));
    pack_ops_kernel<<<dim3(48, (unsigned)n), 256, 0, st>>>(tab);
    MN_LAUNCH_CHECK(ctx);
    ctx->pack_ops.clear();
    return MN_OK;
}

extern "C" {

int mn_abi_version(void) { return MN_ABI_VERSION; }

int mn_debug_tp_program_mode(const mn_model_desc* desc, int mode, unsigned int* table_out, int cap_entries, int* info8) {
    if (!desc || !table_out || !info8 || mode < MN_TP_INFER || mode > MN_TP_DGRAD) return MN_ERR_INVALID;
    if (desc->layers < 1 || desc->layers > MN_MAX_LAYERS || desc->xyz_dim < 3 || desc->xyz_dim > 4 || desc->n_skip < 0 || desc->n_skip > 8)
        return MN_ERR_INVALID;
    mn_model m;
    m.d = *desc;
    build_layout(&m);
    return mn_mlp_tp_program(m, mode, table_out, cap_entries, info8);
}

int mn_debug_tp_program(const mn_model_desc* desc, unsigned int* table_out, int cap_entries, int* info8) {
    return mn_debug_tp_program_mode(desc, MN_TP_INFER, table_out, cap_entries, info8);
}

int mn_create(mn_ctx** out, int device) {
    if (!out) return MN_ERR_INVALID;
    mn_ctx* c = new mn_ctx();
    c->device = device;
    *out = c;
    if (cudaSetDevice(device) != cudaSuccess) {
        c->err = "cudaSetDevice failed (no CUDA device: this library has no CPU fallback)";
        return MN_ERR_CUDA;
    }
    cudaDeviceProp prop;
    MN_CUDA(c, cudaGetDeviceProperties(&prop, device));
    c->sm_count = prop.multiProcessorCount;
    if (prop.major != 9 || prop.minor != 0) {
        c->err = std::string("libmn_b200 is built for sm_90a (Hopper) only; found ") + prop.name;
        return MN_ERR_UNSUPPORTED;
    }
    MN_CUDA(c, cudaMalloc(&c->status_d, sizeof(unsigned int)));
    MN_CUDA(c, cudaMemset(c->status_d, 0, sizeof(unsigned int)));
    return MN_OK;
}

void mn_destroy(mn_ctx* ctx) {
    if (!ctx) return;
    for (cudaEvent_t e : ctx->prof_ev) cudaEventDestroy(e);
    if (ctx->status_d) cudaFree(ctx->status_d);
    if (ctx->pack_ops_d) cudaFree(ctx->pack_ops_d);
    delete ctx;
}

const char* mn_last_error(const mn_ctx* ctx) { return ctx ? ctx->err.c_str() : "null context"; }

int mn_check_status(mn_ctx* ctx, void* stream) {
    if (!ctx) return MN_ERR_INVALID;
    unsigned int h = 0;
    MN_CUDA(ctx, cudaMemcpyAsync(&h, ctx->status_d, sizeof(h), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
    MN_CUDA(ctx, cudaStreamSynchronize((cudaStream_t)stream));
    if (h) MN_CUDA(ctx, cudaMemsetAsync(ctx->status_d, 0, sizeof(h), (cudaStream_t)stream));
    if (h & MN_STATUS_SPHERE)
        return mn_fail(ctx, MN_ERR_SPHERE,
                       "Not all your cameras are bounded by the unit sphere; please make sure the cameras are "
                       "normalized properly!");
    if (h & MN_STATUS_INDEX)
        return mn_fail(ctx, MN_ERR_INVALID, "index out of range (image / pixel index of a ray pair, or row index of a gathered batch)");
    if (h & MN_STATUS_OVERFLOW)
        return mn_fail(ctx, MN_ERR_WORKSPACE, "routing slot capacity exceeded (raise max multiplicity)");
    return MN_OK;
}

long long mn_launch_count(const mn_ctx* ctx) { return ctx ? ctx->launches : 0; }

int mn_profile_enable(mn_ctx* ctx, int on) {
    if (!ctx) return MN_ERR_INVALID;
    ctx->prof_on = on;
    ctx->prof_used = 0;
    return MN_OK;
}

int mn_profile_read(mn_ctx* ctx, double* total_ms, long long* n_launches) {
    if (!ctx) return MN_ERR_INVALID;
    double tot = 0;
    for (size_t i = 0; i + 1 < ctx->prof_used; i += 2) {
        MN_CUDA(ctx, cudaEventSynchronize(ctx->prof_ev[i + 1]));
        float ms = 0;
        MN_CUDA(ctx, cudaEventElapsedTime(&ms, ctx->prof_ev[i], ctx->prof_ev[i + 1]));
        tot += ms;
    }
    if (total_ms) *total_ms = tot;
    if (n_launches) *n_launches = (long long)(ctx->prof_used / 2);
    ctx->prof_used = 0;
    return MN_OK;
}

int mn_model_create(mn_ctx* ctx, const mn_model_desc* desc, mn_model** out) {
    if (!ctx || !desc || !out) return MN_ERR_INVALID;
    const mn_model_desc& d = *desc;
    if (d.kind < 0 || d.kind > 2 || d.n_sub < 1 || d.n_sub > MN_MAX_SUB)
        return mn_fail(ctx, MN_ERR_INVALID, "mn_model_create: kind / n_sub out of range (n_sub <= 64)");
    if (d.layers < 1 || d.layers > MN_MAX_LAYERS || d.xyz_dim < 3 || d.xyz_dim > 4 || d.n_skip < 0 || d.n_skip > 8)
        return mn_fail(ctx, MN_ERR_INVALID, "mn_model_create: layers / xyz_dim / skip_layers out of range");
    if (d.rgb_dim > 3 && d.pos_dir_dim != 0)
        return mn_fail(ctx, MN_ERR_INVALID, "rgb_dim > 3 requires pos_dir_dim == 0 (models/nerf.py:52-53)");
    if (d.kind == 1 && d.n_sub != 2) return mn_fail(ctx, MN_ERR_INVALID, "Cascade needs exactly 2 sub-modules");
    if (d.kind == 2 && d.boundary_margin < 1.0f)
        return mn_fail(ctx, MN_ERR_INVALID, "boundary_margin must be >= 1 (models/mega_nerf.py:11)");
    mn_model* m = new mn_model();
    m->ctx = ctx;
    m->d = d;
    build_layout(m);
    // sub-modules per sample the slot capacity is sized for: 1 under hard routing; with blending a regular centroid grid
    // puts at most 4 (2-D clustering) / 8 (3-D) cells within boundary_margin x d_min for any margin < 2.2 (the nearest cell
    // of the next ring is 2.2 x further than the corner-sharing ones).  mn_model_set_max_multiplicity raises it for other
    // layouts; exceeding it poisons the affected rows with NaN and sets MN_STATUS_OVERFLOW (never a silent wrong blend).
    {
        const int geo = d.cluster_dim_start == 1 ? 4 : 8;
        m->max_multiplicity = (d.kind == 2 && d.boundary_margin > 1.0f) ? (d.n_sub < geo ? d.n_sub : geo) : 1;
        if (d.kind == 2 && d.boundary_margin >= 2.2f) m->max_multiplicity = d.n_sub;
    }
    *out = m;
    MN_CUDA(ctx, cudaMalloc(&m->packed, (size_t)d.n_sub * m->lay.total * sizeof(float)));
    MN_CUDA(ctx, cudaMemset(m->packed, 0, (size_t)d.n_sub * m->lay.total * sizeof(float)));
    MN_CUDA(ctx, cudaMalloc(&m->packed_bwd, (size_t)d.n_sub * m->blay.total * sizeof(float)));
    MN_CUDA(ctx, cudaMemset(m->packed_bwd, 0, (size_t)d.n_sub * m->blay.total * sizeof(float)));
    MN_CUDA(ctx, cudaMalloc(&m->centroids_d, (size_t)MN_MAX_SUB * 3 * sizeof(float)));
    MN_CUDA(ctx, cudaMalloc(&m->counters_d, CNT_TOTAL * sizeof(int)));
    MN_CUDA(ctx, cudaMemset(m->counters_d, 0, CNT_TOTAL * sizeof(int)));
    return MN_OK;
}

void mn_model_destroy(mn_model* m) {
    if (!m) return;
    if (m->packed) cudaFree(m->packed);
    if (m->packed_bwd) cudaFree(m->packed_bwd);
    if (m->centroids_d) cudaFree(m->centroids_d);
    if (m->counters_d) cudaFree(m->counters_d);
    if (m->tc_packed) cudaFree(m->tc_packed);
    if (m->tc_dgrad) cudaFree(m->tc_dgrad);
    if (m->repack_ops) cudaFree(m->repack_ops);
    if (m->repack_first) cudaFree(m->repack_first);
    for (void* p : m->repack_retired) cudaFree(p);
    delete m;
}

int mn_model_set_max_multiplicity(mn_model* m, int mult) {
    if (!m || mult < 1) return MN_ERR_INVALID;
    m->max_multiplicity = mult > m->d.n_sub ? m->d.n_sub : mult;
    return MN_OK;
}

int mn_model_set_centroids(mn_model* m, const float* centroids_d, void* stream) {
    if (!m || !centroids_d) return MN_ERR_INVALID;
    mn_ctx* ctx = m->ctx;
    MN_CUDA(ctx, cudaMemcpyAsync(m->centroids_d, centroids_d, (size_t)m->d.n_sub * 3 * sizeof(float),
                                 cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    return MN_OK;
}

}  // extern "C"

// Queues the fp32 re-layouts of sub-module `sub` from the tensors of *w (ctx->pack_ops): the forward layouts and the data-gradient
// images.  The fp16 tensor-core images (mn_mlp_tc_pack) read the forward layouts, so they go in a second launch.
static int queue_weight_ops(mn_ctx* ctx, mn_model* m, int sub, const mn_nerf_weights* w) {
    const NetDims& nd = m->nd;
    const PackedLayout& l = m->lay;
    float* P = m->packed + (size_t)sub * l.total;
    auto copy = [&](float* dst, const float* src, size_t n) -> int {
        if (!src) return mn_fail(ctx, MN_ERR_INVALID, "mn_model_set_weights: missing tensor");
        PackOp op{src, dst, nullptr, (long long)n, PK_COPY, {0, 0, 0, 0, 0, 0, 0}};
        mn_pack_push(ctx, op);
        return MN_OK;
    };
    int rc;
    for (int i = 0; i < nd.layers; ++i) {
        if (!w->xyz_w[i] || !w->xyz_b[i]) return mn_fail(ctx, MN_ERR_INVALID, "mn_model_set_weights: missing trunk layer");
        pack_T(ctx, w->xyz_w[i], nd.L, l.kin[i], P + l.w[i]);
        if ((rc = copy(P + l.b[i], w->xyz_b[i], nd.L))) return rc;
    }
    if ((rc = copy(P + l.sigma_w, w->sigma_w, nd.L))) return rc;
    if ((rc = copy(P + l.sigma_b, w->sigma_b, 1))) return rc;
    if (nd.has_dir_a) {
        if (!w->final_w || !w->dir_a_w) return mn_fail(ctx, MN_ERR_INVALID, "mn_model_set_weights: missing head");
        pack_T(ctx, w->final_w, nd.L, nd.L, P + l.final_w);
        if ((rc = copy(P + l.final_b, w->final_b, nd.L))) return rc;
        pack_T(ctx, w->dir_a_w, nd.L / 2, nd.L + nd.aux, P + l.dira_w);
        if ((rc = copy(P + l.dira_b, w->dir_a_b, nd.L / 2))) return rc;
    }
    if (!w->rgb_w) return mn_fail(ctx, MN_ERR_INVALID, "mn_model_set_weights: missing rgb head");
    pack_T(ctx, w->rgb_w, nd.rgb_dim, nd.rgb_in, P + l.rgb_w);
    if ((rc = copy(P + l.rgb_b, w->rgb_b, nd.rgb_dim))) return rc;
    if (nd.app > 0)
        if ((rc = copy(P + l.emb, w->embedding_a, (size_t)nd.app_count * nd.app))) return rc;
    if (nd.affine) {
        if (!w->affine_w) return mn_fail(ctx, MN_ERR_INVALID, "mn_model_set_weights: missing affine");
        pack_T(ctx, w->affine_w, 12, nd.app, P + l.aff_w);
        if ((rc = copy(P + l.aff_b, w->affine_b, 12))) return rc;
    }
    // data-gradient images (BwdLayout): the input columns that carry a gradient, in nn.Linear [out][in] order
    {
        const BwdLayout& bl = m->blay;
        float* Q = m->packed_bwd + (size_t)sub * bl.total;
        for (int i = 1; i < nd.layers; ++i) pack_sub(ctx, w->xyz_w[i], nd.L, l.kin[i], l.kin[i] - nd.L, nd.L, Q + bl.w[i]);
        if (nd.has_dir_a) {
            pack_sub(ctx, w->final_w, nd.L, nd.L, 0, nd.L, Q + bl.final_w);
            pack_sub(ctx, w->dir_a_w, nd.L / 2, nd.L + nd.aux, 0, nd.L, Q + bl.dira_f);
            if (nd.app_in_dira) pack_sub(ctx, w->dir_a_w, nd.L / 2, nd.L + nd.aux, nd.L + nd.in_dir, nd.app, Q + bl.dira_e);
        }
    }
    return MN_OK;
}

// The resident table of mn_model_repack from the bound re-layouts of every sub-module (host work and a synchronous upload).
static int upload_repack_table(mn_ctx* ctx, mn_model* m) {
    std::vector<PackOp> ops;
    std::vector<long long> first;
    int n_ops[2];
    long long n_chunks[2];
    for (int k = 0; k < 2; ++k) {
        long long chunks = 0;
        const size_t n0 = ops.size();
        for (const auto& sub_ops : m->bound_ops[k])
            for (const PackOp& op : sub_ops) {
                ops.push_back(op);
                first.push_back(chunks);
                chunks += mn_cdiv(op.count, kRepackChunk);
            }
        first.push_back(chunks);
        n_ops[k] = (int)(ops.size() - n0);
        n_chunks[k] = chunks;
    }
    // A graph captured earlier holds the current table as kernel arguments: an identical table is kept, a different one goes to a
    // new allocation and the old one stays allocated (retired) until the model is destroyed.
    if (m->repack_ops && ops.size() == m->repack_host_ops.size() && first == m->repack_host_first &&
        (ops.empty() || !memcmp(ops.data(), m->repack_host_ops.data(), ops.size() * sizeof(PackOp))))
        return MN_OK;
    PackOp* ops_d = nullptr;
    long long* first_d = nullptr;
    MN_CUDA(ctx, cudaMalloc(&ops_d, (ops.size() > 0 ? ops.size() : 1) * sizeof(PackOp)));
    const cudaError_t e = cudaMalloc(&first_d, first.size() * sizeof(long long));
    if (e != cudaSuccess) { cudaFree(ops_d); MN_CUDA(ctx, e); }
    if (!ops.empty()) MN_CUDA(ctx, cudaMemcpy(ops_d, ops.data(), ops.size() * sizeof(PackOp), cudaMemcpyHostToDevice));
    MN_CUDA(ctx, cudaMemcpy(first_d, first.data(), first.size() * sizeof(long long), cudaMemcpyHostToDevice));
    if (m->repack_ops) {
        m->repack_retired.push_back(m->repack_ops);
        m->repack_retired.push_back(m->repack_first);
    }
    m->repack_ops = ops_d;
    m->repack_first = first_d;
    m->repack_host_ops.swap(ops);
    m->repack_host_first.swap(first);
    for (int k = 0; k < 2; ++k) {
        m->repack_n[k] = n_ops[k];
        m->repack_chunks[k] = n_chunks[k];
    }
    return MN_OK;
}

extern "C" {

int mn_model_set_weights(mn_model* m, int sub, const mn_nerf_weights* w, void* stream) {
    if (!m || !w || sub < 0 || sub >= m->d.n_sub) return MN_ERR_INVALID;
    mn_ctx* ctx = m->ctx;
    cudaStream_t st = (cudaStream_t)stream;
    ctx->pack_ops.clear();
    int rc;
    if ((rc = queue_weight_ops(ctx, m, sub, w))) return rc;
    // launch 1: the fp32 layouts; launch 2 (queued by mn_mlp_tc_pack): the fp16 images that read them
    if ((rc = mn_pack_flush(ctx, st))) return rc;
    if ((rc = mn_mlp_tc_pack(ctx, m, sub, st))) { ctx->pack_ops.clear(); return rc; }
    return mn_pack_flush(ctx, st);
}

int mn_model_bind_weights(mn_model* m, int sub, const mn_nerf_weights* w) {
    if (!m || !w || sub < 0 || sub >= m->d.n_sub) return MN_ERR_INVALID;
    mn_ctx* ctx = m->ctx;
    // Every image the repack writes must exist before its re-layouts are recorded: the forward images are allocated by the first
    // mn_mlp_tc_pack below (on the legacy stream, which orders it after the caller's work).  The transposed images of the
    // tensor-core backward are covered iff they exist, i.e. after a first recording call on the tensor cores: a network trained
    // in fp32 never holds them.
    MN_CUDA(ctx, cudaDeviceSynchronize());
    ctx->pack_ops.clear();
    int rc;
    if ((rc = queue_weight_ops(ctx, m, sub, w))) { ctx->pack_ops.clear(); return rc; }
    std::vector<PackOp> f32_ops;
    f32_ops.swap(ctx->pack_ops);
    if ((rc = mn_mlp_tc_pack(ctx, m, sub, 0))) { ctx->pack_ops.clear(); return rc; }
    std::vector<PackOp> f16_ops;
    f16_ops.swap(ctx->pack_ops);
    MN_CUDA(ctx, cudaStreamSynchronize(0));
    const int n_sub = m->d.n_sub;
    for (int k = 0; k < 2; ++k) m->bound_ops[k].resize(n_sub);
    m->bound.resize(n_sub, 0);
    m->bound_ops[0][sub].swap(f32_ops);
    m->bound_ops[1][sub].swap(f16_ops);
    m->bound[sub] = 1;
    m->bound_dgrad.resize(n_sub, 0);
    m->bound_dgrad[sub] = m->tc_dgrad != nullptr;
    for (int s = 0; s < n_sub; ++s)
        if (!m->bound[s]) return MN_OK;     // the table is built once every sub-module is bound
    return upload_repack_table(ctx, m);
}

int mn_model_repack(mn_ctx* ctx, mn_model* m, void* stream) {
    if (!ctx || !m) return MN_ERR_INVALID;
    if (!m->repack_ops) return mn_fail(ctx, MN_ERR_INVALID, "mn_model_repack: bind the weights of every sub-module first (mn_model_bind_weights)");
    for (char with : m->bound_dgrad)
        if (m->tc_dgrad && !with)
            return mn_fail(ctx, MN_ERR_INVALID, "mn_model_repack: the transposed images of the tensor-core backward were allocated "
                                                "after the weights were bound (a first recording call on the tensor cores): bind again");
    cudaStream_t st = (cudaStream_t)stream;
    // launch 0: the fp32 layouts; launch 1: the fp16 images (forward and data-gradient) that read them
    for (int k = 0, off = 0; k < 2; off += m->repack_n[k] + 1, ++k) {
        if (m->repack_chunks[k] == 0) continue;
        const int op0 = k == 0 ? 0 : m->repack_n[0];
        repack_kernel<<<(unsigned)m->repack_chunks[k], 256, 0, st>>>(m->repack_ops + op0, m->repack_first + off, m->repack_n[k]);
        MN_LAUNCH_CHECK(ctx);
    }
    return MN_OK;
}

size_t mn_debug_weight_images(const mn_model* m, int which, void* dst, size_t cap, void* stream) {
    if (!m || which < 0 || which > 3) return 0;
    const size_t n_sub = (size_t)m->d.n_sub;
    const void* src[4] = {m->packed, m->packed_bwd, m->tc_packed, m->tc_dgrad};
    const size_t bytes[4] = {n_sub * m->lay.total * sizeof(float), n_sub * m->blay.total * sizeof(float),
                             n_sub * (size_t)m->tc.P.sub_bytes, n_sub * (size_t)m->tc.D.sub_bytes};
    if (!src[which]) return 0;
    if (dst && cudaMemcpyAsync(dst, src[which], bytes[which] < cap ? bytes[which] : cap, cudaMemcpyDeviceToDevice,
                               (cudaStream_t)stream) != cudaSuccess) {
        mn_fail(m->ctx, MN_ERR_CUDA, "mn_debug_weight_images: copy failed");
        return 0;
    }
    return bytes[which];
}

// mult: sub-modules per row the slots are sized for; 0 = the model's max_multiplicity
static int64_t slot_capacity(const mn_model* m, int64_t B, int mult = 0) {
    if (m->d.kind != 2) return mn_cdiv(B, MN_BUCKET) * MN_BUCKET;
    return mn_cdiv(B * (mult > 0 ? mult : m->max_multiplicity), MN_BUCKET) * MN_BUCKET + (int64_t)m->d.n_sub * MN_BUCKET;
}

static size_t forward_workspace_bytes(const mn_model* m, int64_t B, int precision, int mult) {
    const int64_t cap = slot_capacity(m, B, mult);
    size_t bytes = 256;
    if (m->d.kind == 2) {
        bytes += mn_align((size_t)cap * sizeof(int));                                       // slot_row
        bytes += mn_align(mn_route_scratch_bytes(m, B));                                    // routing decisions of the count pass
        if (m->d.boundary_margin > 1.0f) {
            bytes += mn_align((size_t)cap * sizeof(float));                                 // slot_w
            bytes += mn_align((size_t)B * m->d.n_sub * sizeof(int));                        // row_slots
            bytes += mn_align((size_t)cap * (m->d.rgb_dim + 1) * sizeof(float));            // slot_out
        }
    }
    if (precision != MN_PREC_FP32) bytes += mn_mlp_tc_workspace(m, cap / MN_TILE, precision);
    return bytes;
}

size_t mn_model_workspace_bytes(const mn_model* m, int64_t B, int precision) {
    return m ? forward_workspace_bytes(m, B, precision, 0) : 0;
}

// Tape header: the routing counters of THIS forward call (the model's own counters are overwritten by the next call).
#define MN_TAPE_HEADER 1024
static_assert(CNT_TOTAL * sizeof(int) <= MN_TAPE_HEADER, "tape header too small");

// Regions of a training tape, in this order: header, slot_row and slot_w (routed models; slot_w only when blending), then
// either the fp32 activation tape or the tensor-core records (encoder tiles, activation images, fp32 head blocks).
struct TapeRegions {
    int* counters;
    int* slot_row;
    float* slot_w;
    float* act;          // fp32 tape
    TrainTcTape tc;      // tensor-core tape
};

// Carves the regions of a tape of `cap` slots at `base` into *r (base may be null when only the size is wanted) and returns the
// tape's size; with_w: routed models keep a slot_w region.
static size_t tape_regions_cap(const mn_model* m, int64_t cap, bool with_w, bool tc, void* base, TapeRegions* r) {
    TapeRegions t{};
    size_t off = 0;
    auto take = [&](size_t n) -> void* {
        void* p = base ? (char*)base + off : nullptr;
        off += mn_align(n);
        return p;
    };
    t.counters = (int*)take(MN_TAPE_HEADER);
    if (m->d.kind == 2) {
        t.slot_row = (int*)take((size_t)cap * sizeof(int));
        if (with_w) t.slot_w = (float*)take((size_t)cap * sizeof(float));
    }
    if (tc) {
        const int64_t n_tiles = cap / MN_TILE;
        t.tc.xreg = (unsigned char*)take((size_t)n_tiles * m->tc.P.x_tile_bytes);
        t.tc.act = (unsigned char*)take((size_t)n_tiles * m->tc.act_tile_bytes);
        t.tc.f32 = (float*)take((size_t)n_tiles * MN_TC_F32_ROWS * MN_TILE * sizeof(float));
    } else {
        const int TM = mn_tape_tm(m->nd.L);
        t.act = (float*)take((size_t)(cap / TM) * m->tape.a_total * TM * sizeof(float));
    }
    if (r) *r = t;
    return off;
}

// The tape of a model call over B rows.
static size_t tape_regions(const mn_model* m, int64_t B, bool tc, void* base, TapeRegions* r = nullptr) {
    return tape_regions_cap(m, slot_capacity(m, B), m->d.boundary_margin > 1.0f, tc, base, r);
}

// The child module's shape error (models/nerf.py:121-123).
static int shape_error(mn_ctx* ctx, int64_t rows, int cols, int expected, int xyz_dim) {
    char buf[256];
    snprintf(buf, sizeof(buf), "Unexpected input shape: torch.Size([%lld, %d]) (expected: %d, xyz_dim: %d)", (long long)rows, cols,
             expected, xyz_dim);
    return mn_fail(ctx, MN_ERR_SHAPE, buf);
}

// What a model call runs: inference at its precision, or a recording forward into the caller's tape - a training call (fp32: the
// fp32 activation tape; tc_f16: the tensor-core records) or the test hook mn_debug_tc_forward_record (tensor-core records of every
// network with a tensor-core forward, trained there or not).
enum CallRun { RUN_INFER, RUN_TRAIN, RUN_TC_HOOK };

// One model call, as its entry point has checked it.
struct ModelCall {
    RowSrc src{};
    int64_t B = 0;                      // rows
    int64_t cap = 0;                    // slots (slot_capacity)
    // How rows become slots.  kind 0 / 1: every row through one sub-module (Cascade: the coarse one when use_coarse).  kind 2: the
    // live rows routed by distance into slots sized for mult sub-modules per row, or, when id_col > 0 (the owner side of an
    // expert-parallel query), bucketed by the sub-module id in payload column id_col (the density noise follows it if has_noise).
    int use_coarse = 0;
    LiveRows live{};
    int mult = 0;
    int id_col = 0, has_noise = 0;
    int sigma_only = 0;
    const float* sigma_noise = nullptr;
    CallRun run = RUN_INFER;
    int precision = MN_PREC_FP32;
    TapeRegions tape{};                 // recording calls: the regions of the caller's tape
    float* out = nullptr;
};

// Runs a checked model call: carves the workspace, builds the slots (a recording call keeps the slot mapping and this call's
// routing counters in its tape), runs the MLP engine and combines blended rows.
static int model_call(mn_ctx* ctx, mn_model* m, const ModelCall& c, void* workspace_d, size_t workspace_bytes, cudaStream_t st) {
    const mn_model_desc& d = m->d;
    const bool record = c.run != RUN_INFER;
    MlpArgs a{};
    a.nd = m->nd;
    a.lay = m->lay;
    a.packed = m->packed;
    a.src = c.src;
    a.n_sub = d.n_sub;
    a.B = c.B;
    a.sigma_only = c.sigma_only;
    a.sigma_noise = c.sigma_noise;
    a.out = c.out;
    a.out_cols = c.sigma_only ? 1 : m->nd.rgb_dim + 1;
    a.live = c.live;

    char* ws = (char*)workspace_d;
    auto carve = [&](size_t n) { char* p = ws; ws += mn_align(n); return p; };
    int rc;
    int* row_slots = nullptr;
    float* slot_out = nullptr;
    if (d.kind == 2) {
        const bool owner = c.id_col > 0;
        const bool blend = !owner && d.boundary_margin > 1.0f;
        // owner training: the tape holds the slot mapping, the workspace the scratch alone, 256 bytes in
        int* slot_row = (int*)carve(owner && record ? 256 : (size_t)c.cap * sizeof(int));
        void* scratch = carve(owner ? mn_route_assigned_scratch_bytes(c.B) : mn_route_scratch_bytes(m, c.B));
        float* slot_w = nullptr;
        if (blend) {
            slot_w = (float*)carve((size_t)c.cap * sizeof(float));
            row_slots = (int*)carve((size_t)c.B * d.n_sub * sizeof(int));
            slot_out = (float*)carve((size_t)c.cap * a.out_cols * sizeof(float));
        }
        if (record) {
            slot_row = c.tape.slot_row;
            slot_w = c.tape.slot_w;
        }
        rc = owner ? mn_route_build_assigned(ctx, m, c.src.x, c.B, c.src.cols, c.id_col, c.has_noise, c.cap, slot_row, scratch,
                                             &a.sigma_noise, st)
                   : mn_route_build(ctx, m, c.src, c.B, c.live, c.cap, slot_row, slot_w, row_slots, scratch, st);
        if (rc) return rc;
        if (record)
            MN_CUDA(ctx, cudaMemcpyAsync(c.tape.counters, m->counters_d, CNT_TOTAL * sizeof(int), cudaMemcpyDeviceToDevice, st));
        a.slot_row = slot_row;
        a.slot_w = slot_w;
        a.counters = m->counters_d;
        a.B = c.cap;
        a.scatter = blend ? 0 : 1;
        if (blend) a.out = slot_out;
    } else {
        a.fixed_sub = (d.kind == 1) ? (c.use_coarse ? 0 : 1) : 0;
        a.scatter = 1;
    }

    a.tape = c.tape.act;       // fp32 recording calls: the activation tape
    if (a.tape) a.tl = m->tape;
    const int64_t n_tiles = c.cap / MN_TILE;
    if (record && c.precision != MN_PREC_FP32)
        rc = mn_mlp_tc_launch_record(ctx, m, a, n_tiles, c.tape.tc, c.run == RUN_TRAIN, st);
    else if (c.precision == MN_PREC_FP32)
        rc = mn_mlp_simt_launch(ctx, a, n_tiles, st);
    else
        rc = mn_mlp_tc_launch(ctx, m, a, n_tiles, c.precision, ws, workspace_bytes - (size_t)(ws - (char*)workspace_d), st);
    if (rc) return rc;
    if (row_slots) return mn_route_combine(ctx, m, c.B, c.live, row_slots, slot_out, a.out_cols, c.out, st);
    return MN_OK;
}

// A model call over mn_rows (c.src.gather: a row gather of ray-structured rows): checks the rows, the workspace and the tape (when
// tape_d is set), then runs it.
static int forward_rows(mn_ctx* ctx, mn_model* m, const mn_rows* rows, ModelCall c, void* workspace_d, size_t workspace_bytes,
                        void* tape_d, size_t tape_bytes, cudaStream_t st) {
    if (!ctx || !m || !rows || c.B < 0) return MN_ERR_INVALID;
    if (c.src.gather && rows->mode != 1) return mn_fail(ctx, MN_ERR_INVALID, "mn_model_forward: a row gather needs ray-structured rows");
    const mn_model_desc& d = m->d;
    const int has_dir = (!c.sigma_only && d.pos_dir_dim > 0) ? 1 : 0;
    const int has_idx = (!c.sigma_only && d.appearance_dim > 0) ? 1 : 0;
    const int prefix = (d.kind == 2 && d.xyz_real) ? 3 : 0;

    RowSrc& src = c.src;
    src.xyz_dim = d.xyz_dim;
    src.net_off = prefix;
    src.x = rows->x_d;
    src.cols = rows->cols;
    if (rows->mode == 0) {
        const int expected = d.xyz_dim + 3 * has_dir + has_idx;
        // the child module is what raises; it sees the row matrix minus the routing prefix, so report that shape.
        if (rows->cols - prefix != expected) return shape_error(ctx, c.B, rows->cols - prefix, expected, d.xyz_dim);
        src.div = 1;
        // nerf.py:146 reads directions as x[:, -4:-1]; :149 the index as x[:, -1]
        src.dirs = rows->x_d + rows->cols - 4;
        src.dir_stride = rows->cols;
        src.idx = rows->x_d + rows->cols - 1;
        src.idx_stride = rows->cols;
        src.dir_quirk = 0;  // the pointer arithmetic above already reproduces the slice
    } else {
        if (rows->cols - prefix != d.xyz_dim)
            return shape_error(ctx, c.B, rows->cols - prefix + 3 * (rows->dirs_d ? 1 : 0) + (rows->idx_d ? 1 : 0),
                               d.xyz_dim + 3 * has_dir + has_idx, d.xyz_dim);
        if ((has_dir && !rows->dirs_d) || (has_idx && !rows->idx_d) || rows->samples_per_ray < 1)
            return mn_fail(ctx, MN_ERR_INVALID, "mn_model_forward: ray-structured rows lack dirs / indices");
        src.div = rows->samples_per_ray;
        src.dirs = rows->dirs_d;
        src.dir_stride = rows->dir_stride;
        src.idx = rows->idx_d;
        src.idx_stride = 1;
        src.dir_quirk = (has_dir && !has_idx) ? 1 : 0;  // [xyz, dir] rows: x[:, -4:-1] = (z, dx, dy)
    }
    if (c.B == 0) return MN_OK;

    c.cap = slot_capacity(m, c.B, c.mult);
    // a recording call runs no tensor-core inference, so its workspace holds none
    const size_t need = forward_workspace_bytes(m, c.B, c.run == RUN_INFER ? c.precision : MN_PREC_FP32, c.mult);
    if (need > 256 && (!workspace_d || workspace_bytes < need))
        return mn_fail(ctx, MN_ERR_WORKSPACE, "mn_model_forward: workspace too small");
    // training forward: the routing tables and the activations outlive the call inside the caller's tape
    if (tape_d && tape_bytes < tape_regions(m, c.B, c.precision != MN_PREC_FP32, tape_d, &c.tape))
        return mn_fail(ctx, MN_ERR_WORKSPACE, "mn_model_forward_train: tape too small");
    return model_call(ctx, m, c, workspace_d, workspace_bytes, st);
}

int mn_model_forward(mn_ctx* ctx, mn_model* m, const mn_rows* rows, int64_t B, int use_coarse, int sigma_only,
                     const float* sigma_noise_d, int precision, float* out_d, void* workspace_d,
                     size_t workspace_bytes, void* stream) {
    ModelCall c;
    c.B = B;
    c.use_coarse = use_coarse;
    c.sigma_only = sigma_only;
    c.sigma_noise = sigma_noise_d;
    c.precision = precision;
    c.out = out_d;
    return forward_rows(ctx, m, rows, c, workspace_d, workspace_bytes, nullptr, 0, (cudaStream_t)stream);
}

// ---- owner side of an expert-parallel query (mega_nerf_b200/expert_parallel.py) ------------------------------------
// Rows arrive with their sub-module id, so the router's bucket count / scan / scatter run on the ids (no distances) and every
// sub-module runs on its bucket in one MLP launch sequence, results scattered back to the rows' own indices.
size_t mn_model_forward_assigned_workspace_bytes(const mn_model* m, int64_t n, int precision) {
    if (!m || n < 0) return 0;
    const int64_t cap = slot_capacity(m, n, 1);
    size_t bytes = 256 + mn_align((size_t)cap * sizeof(int)) + mn_align(mn_route_assigned_scratch_bytes(n));
    if (precision != MN_PREC_FP32) bytes += mn_mlp_tc_workspace(m, cap / MN_TILE, precision);
    return bytes;
}

// The payload rows of an owner call: checks the column count (the child's MN_ERR_SHAPE) and fills the owner fields of *c - the rows,
// the sub-module id column, and the mode-0 RowSrc of `cols` columns inside the wider payload row: directions x[:, -4:-1], image
// index x[:, -1] (nerf.py:146,149).  Every bucketed slot runs through its own sub-module, results scattered to the rows' own indices.
static int assigned_rows(mn_ctx* ctx, const mn_model* m, const float* rows_d, int64_t n, int cols, int has_noise, const char* who,
                         ModelCall* c) {
    if (m->d.kind != 2) return mn_fail(ctx, MN_ERR_INVALID, std::string(who) + ": not a MegaNeRF model");
    const mn_model_desc& d = m->d;
    const int expected = d.xyz_dim + 3 * (d.pos_dir_dim > 0 ? 1 : 0) + (d.appearance_dim > 0 ? 1 : 0);
    if (cols != expected) return shape_error(ctx, n, cols, expected, d.xyz_dim);
    const int stride = cols + 1 + (has_noise ? 1 : 0);
    RowSrc& src = c->src;
    src.xyz_dim = d.xyz_dim;
    src.x = rows_d;
    src.cols = stride;
    src.div = 1;
    src.dirs = rows_d + cols - 4;
    src.dir_stride = stride;
    src.idx = rows_d + cols - 1;
    src.idx_stride = stride;
    c->B = n;
    c->id_col = cols;
    c->has_noise = has_noise;
    return MN_OK;
}

int mn_model_forward_assigned(mn_ctx* ctx, mn_model* m, const float* rows_d, int64_t n, int cols, int has_noise, int precision,
                              float* out_d, void* workspace_d, size_t workspace_bytes, void* stream) {
    if (!ctx || !m || n < 0 || cols < 1) return MN_ERR_INVALID;
    ModelCall c;
    int rc;
    if ((rc = assigned_rows(ctx, m, rows_d, n, cols, has_noise, "mn_model_forward_assigned", &c))) return rc;
    if (n == 0) return MN_OK;
    if (!rows_d || !out_d) return MN_ERR_INVALID;
    if (!workspace_d || workspace_bytes < mn_model_forward_assigned_workspace_bytes(m, n, precision))
        return mn_fail(ctx, MN_ERR_WORKSPACE, "mn_model_forward_assigned: workspace too small");
    c.cap = slot_capacity(m, n, 1);
    c.precision = precision;
    c.out = out_d;
    return model_call(ctx, m, c, workspace_d, workspace_bytes, (cudaStream_t)stream);
}

}  // extern "C"

int mn_model_forward_live(mn_ctx* ctx, mn_model* m, const mn_rows* rows, int64_t B, LiveRows live, int use_coarse, int precision,
                          float* out_d, void* workspace_d, size_t workspace_bytes, cudaStream_t st, const int* gather) {
    ModelCall c;
    c.src.gather = gather;
    c.B = B;
    c.use_coarse = use_coarse;
    c.live = live;
    c.precision = precision;
    c.out = out_d;
    return forward_rows(ctx, m, rows, c, workspace_d, workspace_bytes, nullptr, 0, st);
}

// ---- density grid (scripts/create_octree.py:61-105, 139-162) -------------------------------------------------------
// Rows per slab: a multiple of the reference's 32768-row model_chunk_size, large enough that each slab fills the GPU.
#define MN_GRID_SLAB (1 << 18)
// Largest lattice edge: reso^3 rows fit int64_t and every lattice index converts to fp32 exactly.
#define MN_GRID_MAX_RESO 2097151

namespace {

// xyz [n, 3] of lattice rows r0 .. r0 + n - 1: row r = (i * reso + j) * reso + k, point a = ((idx_a + 0.5) / reso - offset_a) / scale_a,
// each operation one IEEE fp32 rounding, as torch evaluates arange / meshgrid on the CPU (create_octree.py:71-76).
__global__ void __launch_bounds__(256) lattice_kernel(int64_t r0, int64_t n, int reso, float ox, float oy, float oz, float sx,
                                                      float sy, float sz, float* __restrict__ xyz) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const int64_t r = r0 + t;
    const int64_t rr = reso;
    const float fr = (float)reso;
    const int i = (int)(r / (rr * rr)), j = (int)((r / rr) % rr), k = (int)(r % rr);
    xyz[t * 3 + 0] = (((float)i + 0.5f) / fr - ox) / sx;
    xyz[t * 3 + 1] = (((float)j + 0.5f) / fr - oy) / sy;
    xyz[t * 3 + 2] = (((float)k + 0.5f) / fr - oz) / sz;
}

}  // namespace

extern "C" {

size_t mn_model_density_grid_workspace_bytes(const mn_model* m, int precision) {
    if (!m) return 0;
    return mn_align((size_t)MN_GRID_SLAB * 3 * sizeof(float)) + forward_workspace_bytes(m, MN_GRID_SLAB, precision, m->d.n_sub);
}

int mn_model_density_grid(mn_ctx* ctx, mn_model* m, int use_coarse, const float offset[3], const float scale[3], int reso,
                          int64_t row0, int64_t n_rows, int precision, float* sigma_out_d, void* workspace_d,
                          size_t workspace_bytes, void* stream) {
    if (!ctx || !m || !offset || !scale) return MN_ERR_INVALID;
    if (reso < 1 || reso > MN_GRID_MAX_RESO)
        return mn_fail(ctx, MN_ERR_INVALID, "mn_model_density_grid: reso " + std::to_string(reso) + " outside 1.." +
                                                std::to_string(MN_GRID_MAX_RESO));
    for (int a = 0; a < 3; ++a)
        if (!(scale[a] > 0.0f && scale[a] < INFINITY))
            return mn_fail(ctx, MN_ERR_INVALID, "mn_model_density_grid: scale must be positive and finite on every axis");
    const int64_t total = (int64_t)reso * reso * reso;
    if (row0 < 0 || n_rows < 0 || row0 > total || n_rows > total - row0)
        return mn_fail(ctx, MN_ERR_INVALID, "mn_model_density_grid: rows [" + std::to_string(row0) + ", " + std::to_string(row0) + " + " +
                                                std::to_string(n_rows) + ") outside the " + std::to_string(total) + "-row lattice");
    if (m->d.xyz_dim != 3 || (m->d.kind == 2 && m->d.xyz_real))
        return mn_fail(ctx, MN_ERR_UNSUPPORTED,
                       "mn_model_density_grid: the model's rows are not plain xyz (xyz_dim != 3 or a real-xyz routing prefix)");
    if (n_rows == 0) return MN_OK;
    if (!sigma_out_d) return MN_ERR_INVALID;
    if (!workspace_d || workspace_bytes < mn_model_density_grid_workspace_bytes(m, precision))
        return mn_fail(ctx, MN_ERR_WORKSPACE, "mn_model_density_grid: workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    float* pts = (float*)workspace_d;
    const size_t pts_bytes = mn_align((size_t)MN_GRID_SLAB * 3 * sizeof(float));
    mn_rows rows{};
    rows.mode = 0;
    rows.x_d = pts;
    rows.cols = 3;
    ModelCall c;
    c.use_coarse = use_coarse;
    c.sigma_only = 1;
    // a dense box reaches past the centroid hull, where more sub-modules blend than max_multiplicity assumes: size the slots of
    // every slab for all of them
    c.mult = m->d.n_sub;
    c.precision = precision;
    for (int64_t s = 0; s < n_rows; s += MN_GRID_SLAB) {
        const int64_t n = n_rows - s < MN_GRID_SLAB ? n_rows - s : MN_GRID_SLAB;
        lattice_kernel<<<(unsigned)mn_cdiv(n, 256), 256, 0, st>>>(row0 + s, n, reso, offset[0], offset[1], offset[2], scale[0], scale[1],
                                                                   scale[2], pts);
        MN_LAUNCH_CHECK(ctx);
        c.B = n;
        c.out = sigma_out_d + s;
        const int rc = forward_rows(ctx, m, &rows, c, (char*)workspace_d + pts_bytes, workspace_bytes - pts_bytes, nullptr, 0, st);
        if (rc) return rc;
    }
    return MN_OK;
}

// ---- training (SURVEY.md §8f-1) --------------------------------------------------------------------
size_t mn_model_tape_bytes(const mn_model* m, int64_t B) { return m ? tape_regions(m, B, false, nullptr) : 0; }

int mn_model_forward_train(mn_ctx* ctx, mn_model* m, const mn_rows* rows, int64_t B, int use_coarse,
                           const float* sigma_noise_d, float* out_d, void* tape_d, size_t tape_bytes, void* workspace_d,
                           size_t workspace_bytes, void* stream) {
    if (!tape_d) return mn_fail(ctx, MN_ERR_INVALID, "mn_model_forward_train: tape is NULL");
    ModelCall c;
    c.B = B;
    c.use_coarse = use_coarse;
    c.sigma_noise = sigma_noise_d;
    c.run = RUN_TRAIN;
    c.out = out_d;
    return forward_rows(ctx, m, rows, c, workspace_d, workspace_bytes, tape_d, tape_bytes, (cudaStream_t)stream);
}

// Workspace of a backward pass over `cap` slots: the fp32 gradient tape, or what the tensor-core pass carves (tc).
static size_t backward_workspace_bytes(const mn_model* m, int64_t cap, bool tc) {
    if (tc) return 256 + mn_train_tc_backward_workspace(m, cap / MN_TILE);
    const int TM = mn_tape_tm(m->nd.L);
    return 256 + mn_align((size_t)(cap / TM) * m->tape.g_total * TM * sizeof(float));
}

size_t mn_model_backward_workspace_bytes(const mn_model* m, int64_t B) { return m ? backward_workspace_bytes(m, slot_capacity(m, B), false) : 0; }

int64_t mn_model_grad_floats(const mn_model* m) { return m ? (int64_t)m->d.n_sub * m->lay.total : 0; }

int mn_model_param_offsets(const mn_model* m, int64_t* out, int n) {
    if (!m || !out || n < MN_PARAM_OFFSETS) return MN_ERR_INVALID;
    const PackedLayout& l = m->lay;
    int k = 0;
    out[k++] = l.total;
    for (int i = 0; i < MN_MAX_LAYERS; ++i) out[k++] = i < m->nd.layers ? l.w[i] : -1;
    for (int i = 0; i < MN_MAX_LAYERS; ++i) out[k++] = i < m->nd.layers ? l.b[i] : -1;
    out[k++] = l.sigma_w; out[k++] = l.sigma_b;
    out[k++] = l.final_w; out[k++] = l.final_b;
    out[k++] = l.dira_w; out[k++] = l.dira_b;
    out[k++] = l.rgb_w; out[k++] = l.rgb_b;
    out[k++] = l.emb; out[k++] = l.aff_w; out[k++] = l.aff_b;
    return MN_OK;
}

// BwdArgs of a backward pass over B rows and `cap` slots; routed models run the slots their forward pass built (model_backward
// points them at the slot mapping and counters saved in the tape), the others run every row through one sub-module.
static BwdArgs bwd_args(const mn_model* m, int64_t B, int64_t cap, int use_coarse, const float* grad_out_d, float* param_grads_d) {
    const mn_model_desc& d = m->d;
    BwdArgs a{};
    a.nd = m->nd;
    a.lay = m->lay;
    a.blay = m->blay;
    a.packed = m->packed;
    a.packed_bwd = m->packed_bwd;
    a.n_sub = d.n_sub;
    a.B = d.kind == 2 ? cap : B;
    a.grad_out = grad_out_d;
    a.grad_rows = B;
    a.out_cols = m->nd.rgb_dim + 1;
    a.gw = param_grads_d;
    if (d.kind != 2) a.fixed_sub = (d.kind == 1) ? (use_coarse ? 0 : 1) : 0;
    return a;
}

// The backward pass of a recording call over `cap` slots: checks the tape and the workspace, then runs the fp32 kernels or the
// tensor-core pass (tc).  owner: the tape of an owner call, which holds no blend weights.  The tensor-core pass checks its
// workspace itself; owner calls hold it to the size mn_model_backward_assigned_workspace_bytes returns.
static int model_backward(mn_ctx* ctx, mn_model* m, BwdArgs a, int64_t cap, bool owner, bool tc, const void* tape_d,
                          size_t tape_bytes, void* workspace_d, size_t workspace_bytes, const char* who, cudaStream_t st) {
    TapeRegions T;
    if (tape_bytes < tape_regions_cap(m, cap, !owner && m->d.boundary_margin > 1.0f, tc, const_cast<void*>(tape_d), &T))
        return mn_fail(ctx, MN_ERR_WORKSPACE, std::string(who) + ": tape too small");
    if ((owner || !tc) && (!workspace_d || workspace_bytes < backward_workspace_bytes(m, cap, tc)))
        return mn_fail(ctx, MN_ERR_WORKSPACE, std::string(who) + ": workspace too small");
    if (m->d.kind == 2) {
        a.slot_row = T.slot_row;
        a.slot_w = T.slot_w;
        a.counters = T.counters;
    }
    if (tc) return mn_train_tc_backward(ctx, m, a, cap / MN_TILE, T.tc, workspace_d, workspace_bytes, st);
    a.tl = m->tape;
    a.act = T.act;
    a.grad = (float*)workspace_d;
    return mn_mlp_bwd_launch(ctx, a, cap / MN_TILE, st);
}

int mn_model_backward(mn_ctx* ctx, mn_model* m, int64_t B, int use_coarse, const float* grad_out_d, const void* tape_d,
                      size_t tape_bytes, float* param_grads_d, void* workspace_d, size_t workspace_bytes, void* stream) {
    if (!ctx || !m || B < 0 || !grad_out_d || !tape_d || !param_grads_d) return MN_ERR_INVALID;
    if (B == 0) return MN_OK;
    const int64_t cap = slot_capacity(m, B);
    return model_backward(ctx, m, bwd_args(m, B, cap, use_coarse, grad_out_d, param_grads_d), cap, false, false, tape_d, tape_bytes,
                          workspace_d, workspace_bytes, "mn_model_backward", (cudaStream_t)stream);
}

// The layout test hooks' view of the tape of a B-row call: out[0] its size, then the offsets of its regions (-1: absent) - counters,
// slot_row, slot_w, then the fp32 activations, or the tensor-core encoder tiles, activation records and fp32 head blocks (tc).
static_assert(MN_F32L_TAPE_ACT == MN_F32L_TAPE_BYTES + 4 && MN_TCL_TAPE_F32 == MN_TCL_TAPE_BYTES + 6, "tape_layout's order");
static void tape_layout(const mn_model* m, int64_t B, bool tc, int64_t* out) {
    char* const base = (char*)(uintptr_t)4096;      // any non-null base: tape_regions_cap returns pointers base + offset
    TapeRegions T{};
    out[0] = (int64_t)tape_regions(m, B, tc, base, &T);
    const void* const p[] = {T.counters, T.slot_row, T.slot_w, tc ? (const void*)T.tc.xreg : T.act, T.tc.act, T.tc.f32};
    for (int i = 0; i < (tc ? 6 : 4); ++i) out[1 + i] = p[i] ? (int64_t)((const char*)p[i] - base) : -1;
}

int mn_debug_fp32_train_layout(const mn_model* m, int64_t B, int64_t* out, int cap) {
    if (!m || !out || B < 0) return MN_ERR_INVALID;
    if (cap < MN_F32L_COUNT) return MN_ERR_WORKSPACE;
    const int TM = mn_tape_tm(m->nd.L);
    out[MN_F32L_TM] = TM;
    out[MN_F32L_N_TILES] = slot_capacity(m, B) / TM;
    out[MN_F32L_CHUNK_TILES] = MN_WG_CHUNK_TILES;
    tape_layout(m, B, false, out + MN_F32L_TAPE_BYTES);
    out[MN_F32L_BWD_BYTES] = (int64_t)mn_model_backward_workspace_bytes(m, B);
    out[MN_F32L_BWD_GRAD] = 0;                       // mn_model_backward: the gradient tape starts the workspace
    const TapeLayout& t = m->tape;
    const int ch[] = {t.a_pe, t.a_aux, t.a_h, t.a_f, t.a_g, t.a_rgb, t.a_lin, t.a_sig, t.a_id, t.a_total,
                      t.g_z, t.g_final, t.g_dira, t.g_rgb, t.g_sig, t.g_total};
    for (int i = 0; i < (int)(sizeof(ch) / sizeof(ch[0])); ++i) out[MN_F32L_A_PE + i] = ch[i];
    return MN_F32L_COUNT;
}

// ---- tensor-core training path (precision tc_f16 for the recording forward and the backward pass) ----------------
int mn_model_train_tc_supported(const mn_model* m) { return (m && m->tc.train && m->tc_packed) ? 1 : 0; }

size_t mn_model_tape_bytes_tc(const mn_model* m, int64_t B) { return m ? tape_regions(m, B, true, nullptr) : 0; }

int mn_model_forward_train_tc(mn_ctx* ctx, mn_model* m, const mn_rows* rows, int64_t B, int use_coarse,
                              const float* sigma_noise_d, float* out_d, void* tape_d, size_t tape_bytes, void* workspace_d,
                              size_t workspace_bytes, void* stream) {
    if (!tape_d) return mn_fail(ctx, MN_ERR_INVALID, "mn_model_forward_train_tc: tape is NULL");
    if (!mn_model_train_tc_supported(m)) return mn_fail(ctx, MN_ERR_UNSUPPORTED, MN_TC_TRAIN_COVERAGE);
    ModelCall c;
    c.B = B;
    c.use_coarse = use_coarse;
    c.sigma_noise = sigma_noise_d;
    c.run = RUN_TRAIN;
    c.precision = MN_PREC_TC_F16;
    c.out = out_d;
    return forward_rows(ctx, m, rows, c, workspace_d, workspace_bytes, tape_d, tape_bytes, (cudaStream_t)stream);
}

int mn_debug_tc_forward_record(mn_ctx* ctx, mn_model* m, const mn_rows* rows, int64_t B, int use_coarse, const float* sigma_noise_d,
                               float* out_d, void* tape_d, size_t tape_bytes, void* workspace_d, size_t workspace_bytes, void* stream) {
    if (!tape_d) return mn_fail(ctx, MN_ERR_INVALID, "mn_debug_tc_forward_record: tape is NULL");
    ModelCall c;
    c.B = B;
    c.use_coarse = use_coarse;
    c.sigma_noise = sigma_noise_d;
    c.run = RUN_TC_HOOK;
    c.precision = MN_PREC_TC_F16;
    c.out = out_d;
    return forward_rows(ctx, m, rows, c, workspace_d, workspace_bytes, tape_d, tape_bytes, (cudaStream_t)stream);
}

size_t mn_model_backward_workspace_bytes_tc(const mn_model* m, int64_t B) { return m ? backward_workspace_bytes(m, slot_capacity(m, B), true) : 0; }

int mn_debug_tc_train_layout(const mn_model* m, int64_t B, int64_t* out, int cap) {
    if (!m || !out || B < 0) return MN_ERR_INVALID;
    const int64_t n_tiles = slot_capacity(m, B) / MN_TILE;
    const int rc = mn_train_tc_layout(m, n_tiles, out, cap);
    if (rc) return rc;
    out[MN_TCL_N_TILES] = n_tiles;
    tape_layout(m, B, true, out + MN_TCL_TAPE_BYTES);
    out[MN_TCL_BWD_BYTES] = (int64_t)mn_model_backward_workspace_bytes_tc(m, B);
    return MN_TCL_IMG + 2 * (int)out[MN_TCL_N_IMG];
}

int mn_model_backward_tc(mn_ctx* ctx, mn_model* m, int64_t B, int use_coarse, const float* grad_out_d, const void* tape_d,
                         size_t tape_bytes, float* param_grads_d, void* workspace_d, size_t workspace_bytes, void* stream) {
    if (!ctx || !m || B < 0 || !grad_out_d || !tape_d || !param_grads_d) return MN_ERR_INVALID;
    if (B == 0) return MN_OK;
    if (!mn_model_train_tc_supported(m)) return mn_fail(ctx, MN_ERR_UNSUPPORTED, "mn_model_backward_tc: unsupported network shape");
    const int64_t cap = slot_capacity(m, B);
    return model_backward(ctx, m, bwd_args(m, B, cap, use_coarse, grad_out_d, param_grads_d), cap, false, true, tape_d, tape_bytes,
                          workspace_d, workspace_bytes, "mn_model_backward_tc", (cudaStream_t)stream);
}

// ---- training on the owner side of an expert-parallel query ------------------------------------------------------------
// The tape of a recording owner call holds max_pairs pairs, bucketed like mn_model_forward_assigned: slot_capacity(m, max_pairs, 1)
// slots and no slot_w (the blend weights are applied at home).  The rows stay where they arrived; slot_row points into them.
static int assigned_train_prec(mn_ctx* ctx, const mn_model* m, int precision, const char* who) {
    if (precision == MN_PREC_FP32) return MN_OK;
    if (precision != MN_PREC_TC_F16) return mn_fail(ctx, MN_ERR_INVALID, std::string(who) + ": training precision is fp32 or tc_f16");
    if (!mn_model_train_tc_supported(m)) return mn_fail(ctx, MN_ERR_UNSUPPORTED, MN_TC_TRAIN_COVERAGE);
    return MN_OK;
}

size_t mn_model_assigned_tape_bytes(const mn_model* m, int64_t max_pairs, int precision) {
    if (!m || max_pairs < 0) return 0;
    return tape_regions_cap(m, slot_capacity(m, max_pairs, 1), false, precision != MN_PREC_FP32, nullptr, nullptr);
}

size_t mn_model_forward_assigned_train_workspace_bytes(const mn_model* m, int64_t n) {
    if (!m || n < 0) return 0;
    return 256 + mn_align(mn_route_assigned_scratch_bytes(n));
}

int mn_model_forward_assigned_train(mn_ctx* ctx, mn_model* m, const float* rows_d, int64_t n, int cols, int has_noise, int64_t max_pairs,
                                    int precision, float* out_d, void* tape_d, size_t tape_bytes, void* workspace_d, size_t workspace_bytes,
                                    void* stream) {
    if (!ctx || !m || n < 0 || cols < 1 || max_pairs < 0) return MN_ERR_INVALID;
    const char* who = "mn_model_forward_assigned_train";
    ModelCall c;
    int rc;
    if ((rc = assigned_rows(ctx, m, rows_d, n, cols, has_noise, who, &c))) return rc;
    if ((rc = assigned_train_prec(ctx, m, precision, who))) return rc;
    if (n == 0) return MN_OK;
    if (!rows_d || !out_d || !tape_d) return mn_fail(ctx, MN_ERR_INVALID, std::string(who) + ": missing buffer");
    c.cap = slot_capacity(m, max_pairs, 1);
    if (tape_bytes < tape_regions_cap(m, c.cap, false, precision != MN_PREC_FP32, tape_d, &c.tape))
        return mn_fail(ctx, MN_ERR_WORKSPACE, std::string(who) + ": tape too small");
    if (!workspace_d || workspace_bytes < mn_model_forward_assigned_train_workspace_bytes(m, n))
        return mn_fail(ctx, MN_ERR_WORKSPACE, std::string(who) + ": workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    // rows whose pair finds no slot (more pairs than max_pairs: the scatter pass drops them and sets MN_STATUS_OVERFLOW) keep this
    // NaN, as do the empty rows (id -1); every other row is written by the MLP
    MN_CUDA(ctx, cudaMemsetAsync(out_d, 0xFF, (size_t)n * (m->nd.rgb_dim + 1) * sizeof(float), st));
    c.run = RUN_TRAIN;
    c.precision = precision;
    c.out = out_d;
    return model_call(ctx, m, c, workspace_d, workspace_bytes, st);
}

size_t mn_model_backward_assigned_workspace_bytes(const mn_model* m, int64_t max_pairs, int precision) {
    if (!m || max_pairs < 0) return 0;
    return backward_workspace_bytes(m, slot_capacity(m, max_pairs, 1), precision != MN_PREC_FP32);
}

int mn_model_backward_assigned(mn_ctx* ctx, mn_model* m, int64_t n, int64_t max_pairs, int precision, const float* grad_out_d,
                               const void* tape_d, size_t tape_bytes, float* param_grads_d, void* workspace_d, size_t workspace_bytes,
                               void* stream) {
    if (!ctx || !m || n < 0 || max_pairs < 0 || !grad_out_d || !tape_d || !param_grads_d) return MN_ERR_INVALID;
    const char* who = "mn_model_backward_assigned";
    if (m->d.kind != 2) return mn_fail(ctx, MN_ERR_INVALID, std::string(who) + ": not a MegaNeRF model");
    int rc;
    if ((rc = assigned_train_prec(ctx, m, precision, who))) return rc;
    if (n == 0) return MN_OK;
    const int64_t cap = slot_capacity(m, max_pairs, 1);
    return model_backward(ctx, m, bwd_args(m, n, cap, 0, grad_out_d, param_grads_d), cap, true, precision != MN_PREC_FP32, tape_d,
                          tape_bytes, workspace_d, workspace_bytes, who, (cudaStream_t)stream);
}

}  // extern "C"

int mn_model_forward_train_live(mn_ctx* ctx, mn_model* m, const mn_rows* rows, int64_t B, LiveRows live, int use_coarse,
                                const float* sigma_noise_d, int precision, float* out_d, void* tape_d, size_t tape_bytes,
                                void* workspace_d, size_t workspace_bytes, cudaStream_t st, const int* gather) {
    if (!tape_d) return mn_fail(ctx, MN_ERR_INVALID, "mn_model_forward_train: tape is NULL");
    if (precision == MN_PREC_TC_F16 && !mn_model_train_tc_supported(m)) return mn_fail(ctx, MN_ERR_UNSUPPORTED, MN_TC_TRAIN_COVERAGE);
    ModelCall c;
    c.src.gather = gather;
    c.B = B;
    c.use_coarse = use_coarse;
    c.live = live;
    c.sigma_noise = sigma_noise_d;
    c.run = RUN_TRAIN;
    c.precision = precision;
    c.out = out_d;
    return forward_rows(ctx, m, rows, c, workspace_d, workspace_bytes, tape_d, tape_bytes, st);
}

int mn_model_backward_live(mn_ctx* ctx, mn_model* m, int64_t B, LiveRows live, int use_coarse, int precision, const float* grad_out_d,
                           const void* tape_d, size_t tape_bytes, float* param_grads_d, void* workspace_d, size_t workspace_bytes,
                           cudaStream_t st) {
    if (!ctx || !m || B < 0 || !grad_out_d || !tape_d || !param_grads_d) return MN_ERR_INVALID;
    if (B == 0) return MN_OK;
    const bool tc = precision == MN_PREC_TC_F16;
    if (tc && !mn_model_train_tc_supported(m)) return mn_fail(ctx, MN_ERR_UNSUPPORTED, "mn_model_backward_tc: unsupported network shape");
    const int64_t cap = slot_capacity(m, B);
    BwdArgs a = bwd_args(m, B, cap, use_coarse, grad_out_d, param_grads_d);
    a.live = live;
    return model_backward(ctx, m, a, cap, false, tc, tape_d, tape_bytes, workspace_d, workspace_bytes,
                          tc ? "mn_model_backward_tc" : "mn_model_backward", st);
}

extern "C" {

int mn_model_last_stats(mn_ctx* ctx, mn_model* m, int64_t* slots, int64_t* tiles, void* stream) {
    if (!ctx || !m) return MN_ERR_INVALID;
    int h[2] = {0, 0};
    MN_CUDA(ctx, cudaMemcpyAsync(h, m->counters_d + CNT_NSLOTS, 2 * sizeof(int), cudaMemcpyDeviceToHost,
                                 (cudaStream_t)stream));
    MN_CUDA(ctx, cudaStreamSynchronize((cudaStream_t)stream));
    if (slots) *slots = h[1];
    if (tiles) *tiles = h[0] / MN_TILE;
    return MN_OK;
}

}  // extern "C"
