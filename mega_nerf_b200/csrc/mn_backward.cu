// Backward pass of the NeRF MLP stage in the fp32 (CUDA-core) arithmetic of mn_mlp_simt.cu — what
// `loss.backward()` computes through models/nerf.py:115-160 and models/mega_nerf.py:34-49 in the
// reference's training step (runner.py:265).  SURVEY.md §8f-1.
//
// Two kernels over the training tapes (TapeLayout, mn_model.cuh):
//   mlp_bwd_data_kernel   one CTA per tile of TM slots.  Reads the upstream gradient of the (blended)
//                         outputs and the activation tape, walks the network backwards and writes
//                         dL/d(pre-activation) of every Linear to the gradient tape; the appearance
//                         embedding / affine gradients, which are gathers, are accumulated here.
//   mlp_bwd_weight_kernel dW[n][k] = sum over the slots of one sub-module of dZ[n][slot] * X[k][slot]
//                         (and db[n] = sum dZ[n][slot]): a 64x64 register-tiled contraction of the two
//                         tapes per CTA over a chunk of tiles, reduced across chunks with fp32 atomics.
// Activations are channel-major per tile ([channel][TM], a warp's lanes own consecutive slots), the
// same layout the forward kernel keeps in shared memory, so every tape access is a coalesced 128-byte
// line and every weight read is a warp-wide broadcast.
#include "mn_model.cuh"

namespace {

// dX[k][r] = sum_n Wd[n][k] * dZ[n][r]   (+ addw[k] * adds[r])   (masked by hmask[k][r] > 0)
// Wd is [Nred][Kout] row-major (BwdLayout); src / dst are [channels][TM] in shared memory, dst != src.
template <int TM>
__device__ __forceinline__ void dgrad_layer(const float* __restrict__ Wd, int Nred, int Kout, const float* src,
                                            float* dst, const float* __restrict__ addw, const float* adds,
                                            const float* __restrict__ hmask, float* __restrict__ gdst) {
    constexpr int RM = TM / 32;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int cb = 0; cb < Kout; cb += 256) {
        const int k0 = cb + warp * 32;
        if (k0 >= Kout) continue;  // warp-uniform
        float acc[RM][32];
#pragma unroll
        for (int j = 0; j < 32; ++j)
#pragma unroll
            for (int i = 0; i < RM; ++i) acc[i][j] = 0.0f;
#pragma unroll 2
        for (int n = 0; n < Nred; ++n) {
            const float4* wp = reinterpret_cast<const float4*>(Wd + (size_t)n * Kout + k0);
            float a[RM];
#pragma unroll
            for (int i = 0; i < RM; ++i) a[i] = src[n * TM + lane + 32 * i];
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                const float4 w = __ldg(wp + q);
#pragma unroll
                for (int i = 0; i < RM; ++i) {
                    acc[i][4 * q + 0] = fmaf(a[i], w.x, acc[i][4 * q + 0]);
                    acc[i][4 * q + 1] = fmaf(a[i], w.y, acc[i][4 * q + 1]);
                    acc[i][4 * q + 2] = fmaf(a[i], w.z, acc[i][4 * q + 2]);
                    acc[i][4 * q + 3] = fmaf(a[i], w.w, acc[i][4 * q + 3]);
                }
            }
        }
#pragma unroll
        for (int j = 0; j < 32; ++j) {
            const int k = k0 + j;
            const float aw = addw ? __ldg(addw + k) : 0.0f;
#pragma unroll
            for (int i = 0; i < RM; ++i) {
                const int r = lane + 32 * i;
                float v = acc[i][j];
                if (addw) v = fmaf(aw, adds[r], v);
                if (hmask && !(hmask[k * TM + r] > 0.0f)) v = 0.0f;   // ReLU backward: grad * (output > 0)
                dst[k * TM + r] = v;
                if (gdst) gdst[k * TM + r] = v;
            }
        }
    }
}

template <int TM>
__global__ void __launch_bounds__(256, 1) mlp_bwd_data_kernel(const BwdArgs a) {
    extern __shared__ float smem[];
    const NetDims& nd = a.nd;
    const TapeLayout& tl = a.tl;
    const int L = nd.L;
    float* GA = smem;                              // [L][TM]
    float* GB = GA + L * TM;                       // [L][TM]
    float* GO = GB + L * TM;                       // [out_cols][TM] upstream gradient (times the blend weight)
    float* DR = GO + a.out_cols * TM;              // [rgb_dim][TM]  gradient of the rgb Linear output
    float* DS = DR + nd.rgb_dim * TM;              // [TM]           gradient of the sigma pre-activation
    int* ROW = reinterpret_cast<int*>(DS + TM);    // [TM]
    const int tid = threadIdx.x;

    const int64_t slot0 = (int64_t)blockIdx.x * TM;
    const int64_t n_slots = a.counters ? a.counters[CNT_NSLOTS] : a.live.rows(a.B);
    if (slot0 >= n_slots) return;
    int sub = a.fixed_sub;
    if (a.counters) {
        sub = 0;
        while (sub + 1 < a.n_sub && slot0 >= a.counters[CNT_START + sub + 1]) ++sub;
    }
    const float* P = a.packed + (size_t)sub * a.lay.total;
    const float* Q = a.packed_bwd + (size_t)sub * a.blay.total;
    const float* A = a.act + (size_t)blockIdx.x * tl.a_total * TM;
    float* G = a.grad + (size_t)blockIdx.x * tl.g_total * TM;
    float* GW = a.gw + (size_t)sub * a.lay.total;

    if (tid < TM) {
        const int64_t slot = slot0 + tid;
        int64_t row = -1;
        if (slot < n_slots) row = a.slot_row ? (int64_t)a.slot_row[slot] : slot;
        ROW[tid] = (int)row;
        // out[row] = sum over the row's slots of (head output * blend weight)   (mega_nerf.py:46-49)
        const float w = (row >= 0 && a.slot_w) ? a.slot_w[slot] : 1.0f;
        for (int c = 0; c < a.out_cols; ++c)
            GO[c * TM + tid] = row >= 0 ? a.grad_out[row * a.out_cols + c] * w : 0.0f;
    }
    __syncthreads();

    // ---- heads
    if (tid < TM) {
        // sigma = act(pre)   (nerf.py:132-136)
        const float pre = A[tl.a_sig * TM + tid];
        float d;
        if (nd.softplus) {
            const float y = pre - 1.0f;                      // softplus(x - 1, beta 1, threshold 20)
            d = y > 20.0f ? 1.0f : 1.0f / (1.0f + expf(-y));
        } else {
            d = pre > 0.0f ? 1.0f : 0.0f;
        }
        const float ds = ROW[tid] >= 0 ? GO[nd.rgb_dim * TM + tid] * d : 0.0f;
        DS[tid] = ds;
        G[tl.g_sig * TM + tid] = ds;
    }
    for (int it = tid; it < TM * nd.rgb_dim; it += 256) {
        const int r = it % TM, c = it / TM;
        float dv = 0.0f;
        if (ROW[r] >= 0) {
            dv = GO[c * TM + r];
            if (nd.rgb_dim == 3) {                           // rgb = sigmoid(.)   (nerf.py:110,160)
                const float s = A[(tl.a_rgb + c) * TM + r];
                dv = (dv * (1.0f - s)) * s;
            }
        }
        DR[c * TM + r] = dv;
        if (!(nd.affine && nd.app > 0)) G[(tl.g_rgb + c) * TM + r] = dv;
    }
    __syncthreads();
    if (nd.affine && nd.app > 0) {
        // rgb' = A(e) rgb + t(e), [A | t] = affine(e).view(3, 4)   (nerf.py:156-158)
        if (tid < TM) {
            const int r = tid;
            float dl[3] = {0.0f, 0.0f, 0.0f};
            if (ROW[r] >= 0) {
                const int id = (int)A[tl.a_id * TM + r];
                const float* e = P + a.lay.emb + (size_t)id * nd.app;
                const float* aw = P + a.lay.aff_w;           // K-major [app][12]
                float Af[12];
                for (int q = 0; q < 12; ++q) Af[q] = P[a.lay.aff_b + q];
                for (int j = 0; j < nd.app; ++j) {
                    const float ej = e[j];
                    for (int q = 0; q < 12; ++q) Af[q] = fmaf(ej, aw[j * 12 + q], Af[q]);
                }
                const float dv[3] = {DR[0 * TM + r], DR[1 * TM + r], DR[2 * TM + r]};
                const float lin[3] = {A[(tl.a_lin + 0) * TM + r], A[(tl.a_lin + 1) * TM + r], A[(tl.a_lin + 2) * TM + r]};
                float dA[12];
                for (int c = 0; c < 3; ++c) {
                    for (int q = 0; q < 3; ++q) {
                        dA[c * 4 + q] = dv[c] * lin[q];
                        dl[q] = fmaf(Af[c * 4 + q], dv[c], dl[q]);
                    }
                    dA[c * 4 + 3] = dv[c];
                }
                float* gaw = GW + a.lay.aff_w;               // gradient in nn.Linear layout [12][app]
                float* ge = GW + a.lay.emb + (size_t)id * nd.app;
                for (int q = 0; q < 12; ++q) atomicAdd(GW + a.lay.aff_b + q, dA[q]);
                for (int j = 0; j < nd.app; ++j) {
                    const float ej = e[j];
                    float de = 0.0f;
                    for (int q = 0; q < 12; ++q) {
                        atomicAdd(gaw + q * nd.app + j, dA[q] * ej);
                        de = fmaf(dA[q], aw[j * 12 + q], de);
                    }
                    atomicAdd(ge + j, de);
                }
            }
            for (int q = 0; q < 3; ++q) {
                DR[q * TM + r] = dl[q];
                G[(tl.g_rgb + q) * TM + r] = dl[q];
            }
        }
        __syncthreads();
    }

    // ---- rgb Linear: d src[k][r] = sum_c W_rgb[c][k] * DR[c][r]   (P + rgb_w is K-major [k][rgb_dim])
    const float* wr = P + a.lay.rgb_w;
    const float* hlast = A + (size_t)(tl.a_h + (nd.layers - 1) * L) * TM;
    float* gz_last = G + (size_t)(tl.g_z + (nd.layers - 1) * L) * TM;
    if (nd.has_dir_a) {
        const float* g = A + (size_t)tl.a_g * TM;            // ReLU output of dir_a_encoding
        for (int it = tid; it < TM * (L / 2); it += 256) {
            const int r = it % TM, k = it / TM;
            float acc = 0.0f;
            for (int c = 0; c < nd.rgb_dim; ++c) acc = fmaf(__ldg(wr + k * nd.rgb_dim + c), DR[c * TM + r], acc);
            const float v = g[k * TM + r] > 0.0f ? acc : 0.0f;
            GA[k * TM + r] = v;
            G[(size_t)(tl.g_dira + k) * TM + r] = v;
        }
        __syncthreads();
        // dir_a_encoding, feature columns -> gradient of xyz_encoding_final's output (no activation, nerf.py:142)
        dgrad_layer<TM>(Q + a.blay.dira_f, L / 2, L, GA, GB, nullptr, nullptr, nullptr, G + (size_t)tl.g_final * TM);
        // dir_a_encoding, appearance-embedding columns -> embedding_a.weight[id]   (nerf.py:148-149)
        if (nd.app_in_dira) {
            const float* we = Q + a.blay.dira_e;             // [L/2][app]
            for (int it = tid; it < TM * nd.app; it += 256) {
                const int r = it % TM, j = it / TM;
                if (ROW[r] < 0) continue;
                float acc = 0.0f;
                for (int n = 0; n < L / 2; ++n) acc = fmaf(__ldg(we + n * nd.app + j), GA[n * TM + r], acc);
                const int id = (int)A[tl.a_id * TM + r];
                atomicAdd(GW + a.lay.emb + (size_t)id * nd.app + j, acc);
            }
        }
        __syncthreads();
        // xyz_encoding_final -> last trunk activation, plus the sigma head, through the last ReLU
        dgrad_layer<TM>(Q + a.blay.final_w, L, L, GB, GA, P + a.lay.sigma_w, DS, hlast, gz_last);
    } else {
        const float* ws = P + a.lay.sigma_w;
        for (int it = tid; it < TM * L; it += 256) {
            const int r = it % TM, k = it / TM;
            float acc = 0.0f;
            for (int c = 0; c < nd.rgb_dim; ++c) acc = fmaf(__ldg(wr + k * nd.rgb_dim + c), DR[c * TM + r], acc);
            acc = fmaf(__ldg(ws + k), DS[r], acc);
            const float v = hlast[k * TM + r] > 0.0f ? acc : 0.0f;
            GA[k * TM + r] = v;
            gz_last[k * TM + r] = v;
        }
    }
    __syncthreads();

    // ---- trunk, last layer first (nerf.py:126-130); layer 0's input is the positional encoding (no gradient)
    float* cur = GA;
    float* other = GB;
    for (int i = nd.layers - 1; i >= 1; --i) {
        const float* hprev = A + (size_t)(tl.a_h + (i - 1) * L) * TM;
        dgrad_layer<TM>(Q + a.blay.w[i], L, L, cur, other, nullptr, nullptr, hprev, G + (size_t)(tl.g_z + (i - 1) * L) * TM);
        float* t = cur;
        cur = other;
        other = t;
        __syncthreads();
    }
}

template <int TM>
size_t bwd_smem_bytes(const NetDims& nd, int out_cols) {
    return (size_t)(2 * nd.L + out_cols + nd.rgb_dim + 1) * TM * 4 + (size_t)TM * 4;
}

// ------------------------------------------------------------------------------------------------
// weight gradients
// ------------------------------------------------------------------------------------------------
#define MN_WG_MAX_OPS (MN_MAX_LAYERS + 4)
struct WOp {
    int dz, N;            // gradient-tape channel of dZ, number of output features
    int xa, ka, xb, kb;   // the Linear's input = two runs of activation-tape channels (second may be empty)
    int w_off, b_off;     // offsets of weight [N][ka+kb] and bias [N] inside one sub-module's gradient block
};
struct WgradArgs {
    WOp op[MN_WG_MAX_OPS];
    int blk_start[MN_WG_MAX_OPS + 1];   // prefix sums of (n blocks x k blocks) per op
    int n_ops;
    TapeLayout tl;
    const float* act;
    const float* grad;
    float* gw;
    int64_t sub_stride;                 // lay.total
    const int* counters;                // saved routing counters or NULL
    int fixed_sub;
    int64_t B;                          // rows when counters == NULL
    LiveRows live;                      // of the B rows when counters == NULL: the tiles past live.rows(B) hold no tape
    int chunk_tiles;
};

template <int TM>
__global__ void __launch_bounds__(256) mlp_bwd_weight_kernel(const WgradArgs a) {
    __shared__ float DZs[64][TM + 1];
    __shared__ float Xs[64][TM + 1];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    int o = 0;
    while (o + 1 < a.n_ops && (int)blockIdx.y >= a.blk_start[o + 1]) ++o;
    const WOp op = a.op[o];
    const int K = op.ka + op.kb;
    const int kblocks = (K + 63) / 64;
    const int local = (int)blockIdx.y - a.blk_start[o];
    const int n0 = (local / kblocks) * 64, k0 = (local % kblocks) * 64;

    int sub = a.fixed_sub;
    int64_t t_lo = 0, t_hi = (a.live.rows(a.B) + TM - 1) / TM;
    if (a.counters) {
        sub = (int)blockIdx.z;
        t_lo = a.counters[CNT_START + sub] / TM;
        t_hi = a.counters[CNT_START + sub + 1] / TM;
    }
    const int64_t t_begin = t_lo + (int64_t)blockIdx.x * a.chunk_tiles;
    const int64_t t_end = min(t_hi, t_begin + (int64_t)a.chunk_tiles);
    if (t_begin >= t_end) return;

    float acc[4][4];
    float bsum[4] = {0.0f, 0.0f, 0.0f, 0.0f};
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.0f;

    for (int64_t t = t_begin; t < t_end; ++t) {
        const float* Gt = a.grad + (size_t)t * a.tl.g_total * TM;
        const float* At = a.act + (size_t)t * a.tl.a_total * TM;
        for (int it = tid; it < 64 * TM; it += 256) {
            const int c = it / TM, r = it % TM;
            const int n = n0 + c, k = k0 + c;
            DZs[c][r] = n < op.N ? Gt[(size_t)(op.dz + n) * TM + r] : 0.0f;
            float x = 0.0f;
            if (k < op.ka) x = At[(size_t)(op.xa + k) * TM + r];
            else if (k < K) x = At[(size_t)(op.xb + (k - op.ka)) * TM + r];
            Xs[c][r] = x;
        }
        __syncthreads();
#pragma unroll 4
        for (int r = 0; r < TM; ++r) {
            float dz[4], x[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) dz[i] = DZs[ty * 4 + i][r];
#pragma unroll
            for (int j = 0; j < 4; ++j) x[j] = Xs[tx + 16 * j][r];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                bsum[i] += dz[i];
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(dz[i], x[j], acc[i][j]);
            }
        }
        __syncthreads();
    }

    float* W = a.gw + (size_t)sub * a.sub_stride;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int n = n0 + ty * 4 + i;
        if (n >= op.N) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int k = k0 + tx + 16 * j;
            if (k < K) atomicAdd(W + op.w_off + (size_t)n * K + k, acc[i][j]);
        }
        if (k0 == 0 && tx == 0 && op.b_off >= 0) atomicAdd(W + op.b_off + n, bsum[i]);
    }
}

}  // namespace

int mn_mlp_bwd_launch(mn_ctx* ctx, const BwdArgs& a, int64_t n_tiles128, cudaStream_t st) {
    const NetDims& nd = a.nd;
    const TapeLayout& tl = a.tl;
    if (nd.L % 64 != 0 || nd.L > 512 || nd.L < 64)
        return mn_fail(ctx, MN_ERR_UNSUPPORTED, "fp32 MLP backward supports layer_dim in {64,...,512} (multiple of 64)");
    if (nd.affine && nd.rgb_dim != 3)
        return mn_fail(ctx, MN_ERR_UNSUPPORTED, "affine appearance needs rgb_dim == 3 (models/nerf.py:156-158)");
    if (n_tiles128 <= 0) return MN_OK;
    const int TM = mn_tape_tm(nd.L);
    const int64_t n_tiles = n_tiles128 * (MN_TILE / TM);

    mn_prof_begin(ctx, st);   // bench.py --mode train: data + weight gradient kernels timed as one span
    // ---- data gradients
    if (TM == 64) {
        const size_t sm = bwd_smem_bytes<64>(nd, a.out_cols);
        MN_CUDA(ctx, cudaFuncSetAttribute(mlp_bwd_data_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
        mlp_bwd_data_kernel<64><<<(unsigned)n_tiles, 256, sm, st>>>(a);
    } else {
        const size_t sm = bwd_smem_bytes<32>(nd, a.out_cols);
        MN_CUDA(ctx, cudaFuncSetAttribute(mlp_bwd_data_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
        mlp_bwd_data_kernel<32><<<(unsigned)n_tiles, 256, sm, st>>>(a);
    }
    MN_LAUNCH_CHECK(ctx);

    // ---- weight gradients: one op per Linear
    WgradArgs w{};
    const int L = nd.L;
    int n = 0;
    auto add = [&](int dz, int N, int xa, int ka, int xb, int kb, int w_off, int b_off) {
        w.op[n] = WOp{dz, N, xa, ka, xb, kb, w_off, b_off};
        ++n;
    };
    for (int i = 0; i < nd.layers; ++i) {
        const int dz = tl.g_z + i * L;
        if (i == 0)
            add(dz, L, tl.a_pe, nd.in_xyz, 0, 0, a.lay.w[i], a.lay.b[i]);
        else if ((nd.skip_mask >> i) & 1)
            add(dz, L, tl.a_pe, nd.in_xyz, tl.a_h + (i - 1) * L, L, a.lay.w[i], a.lay.b[i]);   // cat[PE, h]
        else
            add(dz, L, tl.a_h + (i - 1) * L, L, 0, 0, a.lay.w[i], a.lay.b[i]);
    }
    const int h_last = tl.a_h + (nd.layers - 1) * L;
    add(tl.g_sig, 1, h_last, L, 0, 0, a.lay.sigma_w, a.lay.sigma_b);
    if (nd.has_dir_a) {
        add(tl.g_final, L, h_last, L, 0, 0, a.lay.final_w, a.lay.final_b);
        add(tl.g_dira, L / 2, tl.a_f, L, tl.a_aux, nd.aux, a.lay.dira_w, a.lay.dira_b);   // cat[f, PE_dir, emb_a]
        add(tl.g_rgb, nd.rgb_dim, tl.a_g, L / 2, 0, 0, a.lay.rgb_w, a.lay.rgb_b);
    } else {
        add(tl.g_rgb, nd.rgb_dim, h_last, L, 0, 0, a.lay.rgb_w, a.lay.rgb_b);
    }
    w.n_ops = n;
    int blocks = 0;
    for (int i = 0; i < n; ++i) {
        w.blk_start[i] = blocks;
        blocks += ((w.op[i].N + 63) / 64) * ((w.op[i].ka + w.op[i].kb + 63) / 64);
    }
    w.blk_start[n] = blocks;
    w.tl = tl;
    w.act = a.act;
    w.grad = a.grad;
    w.gw = a.gw;
    w.sub_stride = a.lay.total;
    w.counters = a.counters;
    w.fixed_sub = a.fixed_sub;
    w.B = a.B;
    w.live = a.live;
    w.chunk_tiles = MN_WG_CHUNK_TILES;
    const unsigned gx = (unsigned)mn_cdiv(n_tiles, w.chunk_tiles);
    const dim3 grid(gx, (unsigned)blocks, (unsigned)(a.counters ? a.n_sub : 1));
    if (TM == 64)
        mlp_bwd_weight_kernel<64><<<grid, 256, 0, st>>>(w);
    else
        mlp_bwd_weight_kernel<32><<<grid, 256, 0, st>>>(w);
    mn_prof_end(ctx, st);
    MN_LAUNCH_CHECK(ctx);
    return MN_OK;
}
