// Context / model management and the nn.Module-level forward entry point of the C ABI.
#include <cuda_fp16.h>

#include <vector>

#include "mn_model.cuh"

namespace {

__global__ void __launch_bounds__(256) pack_ops_kernel(const PackOp* __restrict__ ops) {
    const PackOp op = ops[blockIdx.y];
    const float* __restrict__ src = op.src;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < op.count; i += (long long)gridDim.x * blockDim.x) {
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
            case PK_RGBW: {           // K-major Wt[k][c] -> [c][k]
                const int K = op.p[0], Cc = op.p[1];
                reinterpret_cast<float*>(op.dst)[(i % Cc) * K + i / Cc] = src[i];
                break;
            }
        }
    }
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

int mn_debug_tp_program(const mn_model_desc* desc, unsigned int* table_out, int cap_entries, int* info8) {
    if (!desc || !table_out || !info8) return MN_ERR_INVALID;
    if (desc->layers < 1 || desc->layers > MN_MAX_LAYERS || desc->xyz_dim < 3 || desc->xyz_dim > 4 || desc->n_skip < 0 || desc->n_skip > 8)
        return MN_ERR_INVALID;
    mn_model m;
    m.d = *desc;
    build_layout(&m);
    return mn_mlp_tp_program(m, table_out, cap_entries, info8);
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

int mn_model_set_weights(mn_model* m, int sub, const mn_nerf_weights* w, void* stream) {
    if (!m || !w || sub < 0 || sub >= m->d.n_sub) return MN_ERR_INVALID;
    mn_ctx* ctx = m->ctx;
    cudaStream_t st = (cudaStream_t)stream;
    const NetDims& nd = m->nd;
    const PackedLayout& l = m->lay;
    float* P = m->packed + (size_t)sub * l.total;
    ctx->pack_ops.clear();
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
    // launch 1: the fp32 layouts; launch 2 (queued by mn_mlp_tc_pack): the fp16 images that read them
    if ((rc = mn_pack_flush(ctx, st))) return rc;
    if ((rc = mn_mlp_tc_pack(ctx, m, sub, st))) { ctx->pack_ops.clear(); return rc; }
    return mn_pack_flush(ctx, st);
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

// Carves the regions of a tape at `base` into *r (base may be null when only the size is wanted) and returns the tape's size.
static size_t tape_regions(const mn_model* m, int64_t B, bool tc, void* base, TapeRegions* r = nullptr) {
    const int64_t cap = slot_capacity(m, B);
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
        if (m->d.boundary_margin > 1.0f) t.slot_w = (float*)take((size_t)cap * sizeof(float));
    }
    if (tc) {
        const int64_t n_tiles = cap / MN_TILE;
        t.tc.xreg = (unsigned char*)take((size_t)n_tiles * mn_train_tc_x_tile_bytes(m));
        t.tc.act = (unsigned char*)take((size_t)n_tiles * mn_train_tc_act_tile_bytes(m));
        t.tc.f32 = (float*)take((size_t)n_tiles * MN_TC_F32_ROWS * MN_TILE * sizeof(float));
    } else {
        const int TM = mn_tape_tm(m->nd.L);
        t.act = (float*)take((size_t)(cap / TM) * m->tape.a_total * TM * sizeof(float));
    }
    if (r) *r = t;
    return off;
}

// train_tc != 0: recording forward on the tensor cores (precision tc_f16) into the tensor-core tape regions.
// live: the rows that hold data when their count lives on the device (inference only), see LiveRows.
// mult: sub-modules per row the routing slots of this call are sized for (inference only; 0 = the model's max_multiplicity).
static int model_forward_impl(mn_ctx* ctx, mn_model* m, const mn_rows* rows, int64_t B, int use_coarse, int sigma_only,
                              const float* sigma_noise_d, int precision, float* out_d, void* workspace_d,
                              size_t workspace_bytes, void* tape_d, size_t tape_bytes, void* stream, int train_tc = 0,
                              LiveRows live = LiveRows{}, int mult = 0) {
    if (!ctx || !m || !rows || B < 0) return MN_ERR_INVALID;
    const mn_model_desc& d = m->d;
    const NetDims& nd = m->nd;
    cudaStream_t st = (cudaStream_t)stream;
    const int has_dir = (!sigma_only && d.pos_dir_dim > 0) ? 1 : 0;
    const int has_idx = (!sigma_only && d.appearance_dim > 0) ? 1 : 0;
    const int prefix = (d.kind == 2 && d.xyz_real) ? 3 : 0;

    RowSrc src{};
    src.xyz_dim = d.xyz_dim;
    src.net_off = prefix;
    if (rows->mode == 0) {
        const int expected = d.xyz_dim + 3 * has_dir + has_idx;
        if (rows->cols - prefix != expected) {
            char buf[256];
            // the child module is what raises (models/nerf.py:121-123); it sees the row matrix minus the
            // routing prefix, so report that shape.
            snprintf(buf, sizeof(buf), "Unexpected input shape: torch.Size([%lld, %d]) (expected: %d, xyz_dim: %d)",
                     (long long)B, rows->cols - prefix, expected, d.xyz_dim);
            return mn_fail(ctx, MN_ERR_SHAPE, buf);
        }
        src.x = rows->x_d;
        src.cols = rows->cols;
        src.div = 1;
        // nerf.py:146 reads directions as x[:, -4:-1]; :149 the index as x[:, -1]
        src.dirs = rows->x_d + rows->cols - 4;
        src.dir_stride = rows->cols;
        src.idx = rows->x_d + rows->cols - 1;
        src.idx_stride = rows->cols;
        src.dir_quirk = 0;  // the pointer arithmetic above already reproduces the slice
    } else {
        if (rows->cols - prefix != d.xyz_dim) {
            char buf[256];
            snprintf(buf, sizeof(buf), "Unexpected input shape: torch.Size([%lld, %d]) (expected: %d, xyz_dim: %d)",
                     (long long)B, rows->cols - prefix + 3 * (rows->dirs_d ? 1 : 0) + (rows->idx_d ? 1 : 0),
                     d.xyz_dim + 3 * has_dir + has_idx, d.xyz_dim);
            return mn_fail(ctx, MN_ERR_SHAPE, buf);
        }
        if ((has_dir && !rows->dirs_d) || (has_idx && !rows->idx_d) || rows->samples_per_ray < 1)
            return mn_fail(ctx, MN_ERR_INVALID, "mn_model_forward: ray-structured rows lack dirs / indices");
        src.x = rows->x_d;
        src.cols = rows->cols;
        src.div = rows->samples_per_ray;
        src.dirs = rows->dirs_d;
        src.dir_stride = rows->dir_stride;
        src.idx = rows->idx_d;
        src.idx_stride = 1;
        src.dir_quirk = (has_dir && !has_idx) ? 1 : 0;  // [xyz, dir] rows: x[:, -4:-1] = (z, dx, dy)
    }
    if (B == 0) return MN_OK;

    MlpArgs a{};
    a.nd = nd;
    a.lay = m->lay;
    a.packed = m->packed;
    a.src = src;
    a.n_sub = d.n_sub;
    a.B = B;
    a.sigma_only = sigma_only;
    a.sigma_noise = sigma_noise_d;
    a.out = out_d;
    a.out_cols = sigma_only ? 1 : nd.rgb_dim + 1;
    a.live = live;

    const int64_t cap = slot_capacity(m, B, mult);
    const size_t need = forward_workspace_bytes(m, B, precision, mult);
    if (need > 256 && (!workspace_d || workspace_bytes < need))
        return mn_fail(ctx, MN_ERR_WORKSPACE, "mn_model_forward: workspace too small");
    char* ws = (char*)workspace_d;
    auto carve = [&](size_t n) { char* p = ws; ws += mn_align(n); return p; };
    // training forward: the routing tables and the activations outlive the call inside the caller's tape
    TapeRegions T{};
    if (tape_d && tape_bytes < tape_regions(m, B, train_tc != 0, tape_d, &T))
        return mn_fail(ctx, MN_ERR_WORKSPACE, "mn_model_forward_train: tape too small");

    int rc;
    int* row_slots = nullptr;
    float* slot_out = nullptr;
    if (d.kind == 2) {
        int* slot_row = (int*)carve((size_t)cap * sizeof(int));
        void* route_scratch = carve(mn_route_scratch_bytes(m, B));
        float* slot_w = nullptr;
        const bool blend = d.boundary_margin > 1.0f;
        if (blend) {
            slot_w = (float*)carve((size_t)cap * sizeof(float));
            row_slots = (int*)carve((size_t)B * d.n_sub * sizeof(int));
            slot_out = (float*)carve((size_t)cap * a.out_cols * sizeof(float));
        }
        if (tape_d) {
            slot_row = T.slot_row;
            slot_w = T.slot_w;
        }
        if ((rc = mn_route_build(ctx, m, src, B, live, cap, slot_row, slot_w, row_slots, route_scratch, st))) return rc;
        if (tape_d)
            MN_CUDA(ctx, cudaMemcpyAsync(T.counters, m->counters_d, CNT_TOTAL * sizeof(int), cudaMemcpyDeviceToDevice, st));
        a.slot_row = slot_row;
        a.slot_w = slot_w;
        a.counters = m->counters_d;
        a.B = cap;
        a.scatter = blend ? 0 : 1;
        if (blend) a.out = slot_out;
    } else {
        a.fixed_sub = (d.kind == 1) ? (use_coarse ? 0 : 1) : 0;
        a.scatter = 1;
    }

    const int64_t n_tiles = cap / MN_TILE;
    if (tape_d && train_tc) {
        if ((rc = mn_mlp_tc_launch_train(ctx, m, a, n_tiles, T.tc, st))) return rc;
        if (row_slots) return mn_route_combine(ctx, m, B, live, row_slots, slot_out, a.out_cols, out_d, st);
        return MN_OK;
    }
    if (tape_d) {
        a.tape = T.act;
        a.tl = m->tape;
    }
    if (precision == MN_PREC_FP32)
        rc = mn_mlp_simt_launch(ctx, a, n_tiles, st);
    else
        rc = mn_mlp_tc_launch(ctx, m, a, n_tiles, precision, ws, workspace_bytes - (size_t)(ws - (char*)workspace_d), st);
    if (rc) return rc;
    if (row_slots) return mn_route_combine(ctx, m, B, live, row_slots, slot_out, a.out_cols, out_d, st);
    return MN_OK;
}

int mn_model_forward(mn_ctx* ctx, mn_model* m, const mn_rows* rows, int64_t B, int use_coarse, int sigma_only,
                     const float* sigma_noise_d, int precision, float* out_d, void* workspace_d,
                     size_t workspace_bytes, void* stream) {
    return model_forward_impl(ctx, m, rows, B, use_coarse, sigma_only, sigma_noise_d, precision, out_d, workspace_d,
                              workspace_bytes, nullptr, 0, stream);
}

}  // extern "C"

int mn_model_forward_live(mn_ctx* ctx, mn_model* m, const mn_rows* rows, int64_t B, LiveRows live, int use_coarse, int precision,
                          float* out_d, void* workspace_d, size_t workspace_bytes, cudaStream_t st) {
    return model_forward_impl(ctx, m, rows, B, use_coarse, 0, nullptr, precision, out_d, workspace_d, workspace_bytes, nullptr, 0, st,
                              0, live);
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
    for (int64_t s = 0; s < n_rows; s += MN_GRID_SLAB) {
        const int64_t n = n_rows - s < MN_GRID_SLAB ? n_rows - s : MN_GRID_SLAB;
        lattice_kernel<<<(unsigned)mn_cdiv(n, 256), 256, 0, st>>>(row0 + s, n, reso, offset[0], offset[1], offset[2], scale[0], scale[1],
                                                                   scale[2], pts);
        MN_LAUNCH_CHECK(ctx);
        // a dense box reaches past the centroid hull, where more sub-modules blend than max_multiplicity assumes: size this call's
        // slots for all of them
        const int rc = model_forward_impl(ctx, m, &rows, n, use_coarse, 1, nullptr, precision, sigma_out_d + s, (char*)workspace_d + pts_bytes,
                                          workspace_bytes - pts_bytes, nullptr, 0, stream, 0, LiveRows{}, m->d.n_sub);
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
    return model_forward_impl(ctx, m, rows, B, use_coarse, 0, sigma_noise_d, MN_PREC_FP32, out_d, workspace_d,
                              workspace_bytes, tape_d, tape_bytes, stream);
}

size_t mn_model_backward_workspace_bytes(const mn_model* m, int64_t B) {
    if (!m) return 0;
    const int64_t cap = slot_capacity(m, B);
    const int TM = mn_tape_tm(m->nd.L);
    return 256 + mn_align((size_t)(cap / TM) * m->tape.g_total * TM * sizeof(float));
}

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

// BwdArgs fields common to both backward passes; routed models read the slot mapping and counters the forward pass saved
// in the tape, the others run every row through one sub-module.
static BwdArgs bwd_args(const mn_model* m, int64_t B, int use_coarse, const float* grad_out_d, float* param_grads_d,
                        const TapeRegions& T) {
    const mn_model_desc& d = m->d;
    BwdArgs a{};
    a.nd = m->nd;
    a.lay = m->lay;
    a.blay = m->blay;
    a.packed = m->packed;
    a.packed_bwd = m->packed_bwd;
    a.n_sub = d.n_sub;
    a.B = B;
    a.grad_out = grad_out_d;
    a.out_cols = m->nd.rgb_dim + 1;
    a.gw = param_grads_d;
    if (d.kind == 2) {
        a.slot_row = T.slot_row;
        a.slot_w = T.slot_w;
        a.counters = T.counters;
        a.B = slot_capacity(m, B);
    } else {
        a.fixed_sub = (d.kind == 1) ? (use_coarse ? 0 : 1) : 0;
    }
    return a;
}

int mn_model_backward(mn_ctx* ctx, mn_model* m, int64_t B, int use_coarse, const float* grad_out_d, const void* tape_d,
                      size_t tape_bytes, float* param_grads_d, void* workspace_d, size_t workspace_bytes, void* stream) {
    if (!ctx || !m || B < 0 || !grad_out_d || !tape_d || !param_grads_d) return MN_ERR_INVALID;
    if (B == 0) return MN_OK;
    TapeRegions T;
    if (tape_bytes < tape_regions(m, B, false, const_cast<void*>(tape_d), &T))
        return mn_fail(ctx, MN_ERR_WORKSPACE, "mn_model_backward: tape too small");
    if (!workspace_d || workspace_bytes < mn_model_backward_workspace_bytes(m, B))
        return mn_fail(ctx, MN_ERR_WORKSPACE, "mn_model_backward: workspace too small");
    BwdArgs a = bwd_args(m, B, use_coarse, grad_out_d, param_grads_d, T);
    a.tl = m->tape;
    a.act = T.act;
    a.grad = (float*)workspace_d;
    return mn_mlp_bwd_launch(ctx, a, slot_capacity(m, B) / MN_TILE, (cudaStream_t)stream);
}

// ---- tensor-core training path (precision tc_f16 for the recording forward and the backward pass) ----------------
int mn_model_train_tc_supported(const mn_model* m) { return (m && m->train_tc_ok) ? 1 : 0; }

size_t mn_model_tape_bytes_tc(const mn_model* m, int64_t B) { return m ? tape_regions(m, B, true, nullptr) : 0; }

int mn_model_forward_train_tc(mn_ctx* ctx, mn_model* m, const mn_rows* rows, int64_t B, int use_coarse,
                              const float* sigma_noise_d, float* out_d, void* tape_d, size_t tape_bytes, void* workspace_d,
                              size_t workspace_bytes, void* stream) {
    if (!tape_d) return mn_fail(ctx, MN_ERR_INVALID, "mn_model_forward_train_tc: tape is NULL");
    if (!m || !m->train_tc_ok) return mn_fail(ctx, MN_ERR_UNSUPPORTED, MN_TC_TRAIN_COVERAGE);
    return model_forward_impl(ctx, m, rows, B, use_coarse, 0, sigma_noise_d, MN_PREC_FP32, out_d, workspace_d, workspace_bytes, tape_d,
                              tape_bytes, stream, 1);
}

size_t mn_model_backward_workspace_bytes_tc(const mn_model* m, int64_t B) {
    if (!m) return 0;
    return 256 + mn_train_tc_backward_workspace(m, slot_capacity(m, B) / MN_TILE);
}

int mn_model_backward_tc(mn_ctx* ctx, mn_model* m, int64_t B, int use_coarse, const float* grad_out_d, const void* tape_d,
                         size_t tape_bytes, float* param_grads_d, void* workspace_d, size_t workspace_bytes, void* stream) {
    if (!ctx || !m || B < 0 || !grad_out_d || !tape_d || !param_grads_d) return MN_ERR_INVALID;
    if (B == 0) return MN_OK;
    if (!m->train_tc_ok) return mn_fail(ctx, MN_ERR_UNSUPPORTED, "mn_model_backward_tc: unsupported network shape");
    TapeRegions T;
    if (tape_bytes < tape_regions(m, B, true, const_cast<void*>(tape_d), &T))
        return mn_fail(ctx, MN_ERR_WORKSPACE, "mn_model_backward_tc: tape too small");
    BwdArgs a = bwd_args(m, B, use_coarse, grad_out_d, param_grads_d, T);
    a.grad_rows = B;
    return mn_train_tc_backward(ctx, m, a, slot_capacity(m, B) / MN_TILE, T.tc, workspace_d, workspace_bytes, (cudaStream_t)stream);
}

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
