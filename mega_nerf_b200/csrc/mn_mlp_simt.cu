// MN_PREC_FP32: the whole NeRF MLP (models/nerf.py:115-160) for one tile of rows in one CTA, on CUDA
// cores with explicit fp32 FMAs.  This is the parity-mode arithmetic (<= 1e-5 of the fp32 oracle) and
// the on-device cross-check of the tensor-core kernel; activations never leave shared memory.
//
// Layout: activations are kept channel-major in shared memory (act[k][row]) so that a warp's 32 lanes
// own 32 consecutive rows (conflict-free loads/stores) and every weight load is a warp-wide broadcast
// of a contiguous 16-byte chunk of the K-major packed weight matrix.
#include "mn_model.cuh"

namespace {

template <int TM>
__device__ __forceinline__ void gemm_layer(const float* __restrict__ Wt, const float* __restrict__ bias, int N,
                                           const float* s0, int k0, const float* s1, int k1, float* dst,
                                           bool relu, float* __restrict__ gdst = nullptr) {
    constexpr int RM = TM / 32;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int cb = 0; cb < N; cb += 256) {
        const int n0 = cb + warp * 32;
        if (n0 >= N) continue;  // warp-uniform
        float acc[RM][32];
#pragma unroll
        for (int j = 0; j < 32; ++j) {
            const float b = __ldg(bias + n0 + j);
#pragma unroll
            for (int i = 0; i < RM; ++i) acc[i][j] = b;
        }
        int kbase = 0;
#pragma unroll 1
        for (int seg = 0; seg < 2; ++seg) {
            const float* src = seg == 0 ? s0 : s1;
            const int nk = seg == 0 ? k0 : k1;
#pragma unroll 2
            for (int k = 0; k < nk; ++k) {
                const float4* wp = reinterpret_cast<const float4*>(Wt + (size_t)(kbase + k) * N + n0);
                float a[RM];
#pragma unroll
                for (int i = 0; i < RM; ++i) a[i] = src[k * TM + lane + 32 * i];
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
            kbase += nk;
        }
#pragma unroll
        for (int j = 0; j < 32; ++j)
#pragma unroll
            for (int i = 0; i < RM; ++i) {
                float v = acc[i][j];
                if (relu) v = fmaxf(v, 0.0f);
                dst[(n0 + j) * TM + lane + 32 * i] = v;
                if (gdst) gdst[(n0 + j) * TM + lane + 32 * i] = v;   // activation tape (training forward)
            }
    }
}

// Rows of the PE block: the xyz encoding, and later the rgb head's outputs, which can outnumber it (an SH head of degree 4 has
// 75 coefficients, the xyz encoding of pos_xyz_dim 10 has 63 channels).
__host__ __device__ __forceinline__ int simt_pe_rows(const NetDims& nd) { return nd.in_xyz > nd.rgb_dim ? nd.in_xyz : nd.rgb_dim; }

// SAVE = training forward: every value the backward pass needs is also written to the activation tape
// (TapeLayout, mn_model.cuh); the arithmetic is the same instruction stream either way.
template <int TM, bool SAVE>
__global__ void __launch_bounds__(256, 1) mlp_simt_kernel(const MlpArgs a) {
    extern __shared__ float smem[];
    const NetDims& nd = a.nd;
    const int L = nd.L;
    float* const T = SAVE ? a.tape + (size_t)blockIdx.x * a.tl.a_total * TM : nullptr;
    float* PE = smem;                    // [in_xyz][TM]; [simt_pe_rows(nd)] reserved: the rgb head's outputs reuse it
    float* AUX = PE + simt_pe_rows(nd) * TM;    // [aux][TM]  = dir encoding | appearance embedding
    float* H0 = AUX + nd.aux * TM;       // [L][TM]
    float* H1 = H0 + L * TM;             // [L][TM]
    float* SIG = H1 + L * TM;            // [TM]
    int* ROW = reinterpret_cast<int*>(SIG + TM);           // [TM]
    float* XIN = reinterpret_cast<float*>(ROW + TM);       // [TM][8]
    const int tid = threadIdx.x;

    const int64_t slot0 = (int64_t)blockIdx.x * TM;
    const int64_t n_slots = a.n_slots();
    if (slot0 >= n_slots) return;
    int sub = a.fixed_sub;
    if (a.counters) {
        sub = 0;
        while (sub + 1 < a.n_sub && slot0 >= a.counters[CNT_START + sub + 1]) ++sub;
    }
    const float* P = a.packed + (size_t)sub * a.lay.total;

    if (tid < TM) {
        const int64_t slot = slot0 + tid;
        int64_t row = -1;
        if (slot < n_slots) row = a.slot_row ? (int64_t)a.slot_row[slot] : slot;
        ROW[tid] = (int)row;
        float* xi = XIN + tid * 8;
#pragma unroll
        for (int j = 0; j < 8; ++j) xi[j] = 0.0f;
        if (row >= 0) {
            for (int j = 0; j < nd.xyz_dim; ++j) xi[j] = a.src.xyz(row, j);
            if (!a.sigma_only) {
                if (nd.nf_dir > 0)
                    for (int j = 0; j < 3; ++j) xi[4 + j] = a.src.dir(row, j);
                if (nd.app > 0) xi[7] = a.src.index(row);
            }
        }
    }
    __syncthreads();

    // positional encoding of xyz (models/nerf.py:20-25): [x | sin 2^0 x | cos 2^0 x | sin 2^1 x | ...]
    {
        const int per_row = nd.xyz_dim * (1 + nd.nf_xyz);
        for (int it = tid; it < TM * per_row; it += 256) {
            const int r = it % TM, q = it / TM;
            if (q < nd.xyz_dim) {
                PE[q * TM + r] = XIN[r * 8 + q];
            } else {
                const int qq = q - nd.xyz_dim, k = qq / nd.xyz_dim, j = qq % nd.xyz_dim;
                float s, c;
                mn_pe_sincos(XIN[r * 8 + j], k, &s, &c);
                const int base = nd.xyz_dim + k * 2 * nd.xyz_dim;
                PE[(base + j) * TM + r] = s;
                PE[(base + nd.xyz_dim + j) * TM + r] = c;
            }
        }
        if (!a.sigma_only) {
            if (nd.nf_dir > 0) {
                const int per = 3 * (1 + nd.nf_dir);
                for (int it = tid; it < TM * per; it += 256) {
                    const int r = it % TM, q = it / TM;
                    if (q < 3) {
                        AUX[q * TM + r] = XIN[r * 8 + 4 + q];
                    } else {
                        const int qq = q - 3, k = qq / 3, j = qq % 3;
                        float s, c;
                        mn_pe_sincos(XIN[r * 8 + 4 + j], k, &s, &c);
                        AUX[(3 + k * 6 + j) * TM + r] = s;
                        AUX[(3 + k * 6 + 3 + j) * TM + r] = c;
                    }
                }
            }
            if (nd.app_in_dira) {
                const float* emb = P + a.lay.emb;
                for (int it = tid; it < TM * nd.app; it += 256) {
                    const int r = it % TM, j = it / TM;
                    int id = (int)XIN[r * 8 + 7];  // x[:, -1].long()  (nerf.py:149)
                    id = min(max(id, 0), nd.app_count - 1);
                    AUX[(nd.in_dir + j) * TM + r] = emb[(size_t)id * nd.app + j];
                }
            }
        }
    }
    __syncthreads();
    if (SAVE) {
        // PE and AUX are contiguous [channels][TM] blocks in shared memory, same layout as the tape
        for (int it = tid; it < nd.in_xyz * TM; it += 256) T[a.tl.a_pe * TM + it] = PE[it];
        for (int it = tid; it < nd.aux * TM; it += 256) T[a.tl.a_aux * TM + it] = AUX[it];
        if (tid < TM && nd.app > 0) {
            int id = (int)XIN[tid * 8 + 7];
            id = min(max(id, 0), nd.app_count - 1);
            T[a.tl.a_id * TM + tid] = (float)id;
        }
    }

    // trunk (nerf.py:126-130)
    float* cur = nullptr;
    for (int i = 0; i < nd.layers; ++i) {
        float* dst = (i & 1) ? H1 : H0;
        const float* W = P + a.lay.w[i];
        const float* Bv = P + a.lay.b[i];
        float* gd = SAVE ? T + (size_t)(a.tl.a_h + i * L) * TM : nullptr;
        if (i == 0)
            gemm_layer<TM>(W, Bv, L, PE, nd.in_xyz, nullptr, 0, dst, true, gd);
        else if ((nd.skip_mask >> i) & 1)
            gemm_layer<TM>(W, Bv, L, PE, nd.in_xyz, cur, L, dst, true, gd);   // cat[PE, h]  (nerf.py:129)
        else
            gemm_layer<TM>(W, Bv, L, cur, L, nullptr, 0, dst, true, gd);
        cur = dst;
        __syncthreads();
    }
    float* other = (cur == H0) ? H1 : H0;

    // sigma head (nerf.py:132-136)
    if (tid < TM) {
        const float* ws = P + a.lay.sigma_w;
        float acc = P[a.lay.sigma_b];
        for (int k = 0; k < L; ++k) acc = fmaf(cur[k * TM + tid], __ldg(ws + k), acc);
        const int row = ROW[tid];
        if (a.sigma_noise && row >= 0) acc = acc + a.sigma_noise[row];
        if (SAVE) T[a.tl.a_sig * TM + tid] = acc;   // pre-activation (noise included)
        SIG[tid] = nd.softplus ? mn_softplus_shifted(acc) : fmaxf(acc, 0.0f);
    }
    __syncthreads();

    if (a.sigma_only) {
        if (tid < TM) {
            const int row = ROW[tid];
            if (row >= 0) {
                const int64_t o = a.scatter ? (int64_t)row : slot0 + tid;
                float v = SIG[tid];
                if (a.slot_w) v = v * a.slot_w[slot0 + tid];
                a.out[o * a.out_cols] = v;
            }
        }
        return;
    }

    const float* rgb_src = cur;
    if (nd.has_dir_a) {
        // xyz_encoding_final (no activation) then dir_a_encoding + ReLU (nerf.py:141-151)
        gemm_layer<TM>(P + a.lay.final_w, P + a.lay.final_b, L, cur, L, nullptr, 0, other, false,
                       SAVE ? T + (size_t)a.tl.a_f * TM : nullptr);
        __syncthreads();
        gemm_layer<TM>(P + a.lay.dira_w, P + a.lay.dira_b, L / 2, other, L, AUX, nd.aux, cur, true,
                       SAVE ? T + (size_t)a.tl.a_g * TM : nullptr);
        __syncthreads();
        rgb_src = cur;
    }
    // rgb head (nerf.py:152-154)
    float* OUTS = PE;  // [rgb_dim][TM] (simt_pe_rows), PE is dead by now
    {
        const float* wr = P + a.lay.rgb_w;
        const float* br = P + a.lay.rgb_b;
        for (int it = tid; it < TM * nd.rgb_dim; it += 256) {
            const int r = it % TM, c = it / TM;
            float acc = __ldg(br + c);
            for (int k = 0; k < nd.rgb_in; ++k) acc = fmaf(rgb_src[k * TM + r], __ldg(wr + k * nd.rgb_dim + c), acc);
            OUTS[c * TM + r] = acc;
        }
    }
    __syncthreads();
    if (SAVE && tid < TM) {
        // values the backward pass needs: the Linear output of the rgb head (affine models) ...
        if (nd.affine && nd.app > 0)
            for (int c = 0; c < 3; ++c) T[(a.tl.a_lin + c) * TM + tid] = OUTS[c * TM + tid];
    }
    if (tid < TM) {
        const int row = ROW[tid];
        if (SAVE && row < 0)
            for (int c = 0; c < nd.rgb_dim; ++c) T[(a.tl.a_rgb + c) * TM + tid] = 0.0f;
        if (row >= 0) {
            float rgb[3] = {0, 0, 0};
            if (nd.affine && nd.app > 0) {
                // affine appearance (nerf.py:156-158)
                const float* emb = P + a.lay.emb;
                const float* aw = P + a.lay.aff_w;  // [app][12]
                int id = (int)XIN[tid * 8 + 7];
                id = min(max(id, 0), nd.app_count - 1);
                float A[12];
                for (int q = 0; q < 12; ++q) A[q] = P[a.lay.aff_b + q];
                for (int j = 0; j < nd.app; ++j) {
                    const float e = emb[(size_t)id * nd.app + j];
                    for (int q = 0; q < 12; ++q) A[q] = fmaf(e, aw[j * 12 + q], A[q]);
                }
                const float r0 = OUTS[0 * TM + tid], r1 = OUTS[1 * TM + tid], r2 = OUTS[2 * TM + tid];
                for (int c = 0; c < 3; ++c)
                    rgb[c] = fmaf(A[c * 4 + 2], r2, fmaf(A[c * 4 + 1], r1, A[c * 4 + 0] * r0)) + A[c * 4 + 3];
                OUTS[0 * TM + tid] = rgb[0];
                OUTS[1 * TM + tid] = rgb[1];
                OUTS[2 * TM + tid] = rgb[2];
            }
            const int64_t o = (a.scatter ? (int64_t)row : slot0 + tid) * a.out_cols;
            const float w = a.slot_w ? a.slot_w[slot0 + tid] : 1.0f;
            for (int c = 0; c < nd.rgb_dim; ++c) {
                float v = OUTS[c * TM + tid];
                if (nd.rgb_dim == 3) v = mn_sigmoid(v);
                if (SAVE) T[(a.tl.a_rgb + c) * TM + tid] = v;   // ... and the head's output before blending
                a.out[o + c] = a.slot_w ? v * w : v;
            }
            const float s = SIG[tid];
            a.out[o + nd.rgb_dim] = a.slot_w ? s * w : s;
        }
    }
}

template <int TM>
size_t simt_smem_bytes(const NetDims& nd) {
    return (size_t)(simt_pe_rows(nd) + nd.aux + 2 * nd.L + 1) * TM * 4 + (size_t)TM * 4 + (size_t)TM * 8 * 4;
}

}  // namespace

int mn_mlp_simt_launch(mn_ctx* ctx, const MlpArgs& a, int64_t n_tiles128, cudaStream_t st) {
    const NetDims& nd = a.nd;
    if (nd.L % 64 != 0 || nd.L > 512 || nd.L < 64)
        return mn_fail(ctx, MN_ERR_UNSUPPORTED, "fp32 MLP kernel supports layer_dim in {64,...,512} (multiple of 64)");
    if (n_tiles128 <= 0) return MN_OK;
    mn_prof_begin(ctx, st);
    if (a.tape && a.sigma_only) return mn_fail(ctx, MN_ERR_INVALID, "training forward has no sigma_only mode");
#define MN_SIMT_LAUNCH(TM_, SAVE_, MULT_)                                                                            \
    do {                                                                                                             \
        const size_t sm = simt_smem_bytes<TM_>(nd);                                                                  \
        MN_CUDA(ctx, cudaFuncSetAttribute(mlp_simt_kernel<TM_, SAVE_>, cudaFuncAttributeMaxDynamicSharedMemorySize,  \
                                          (int)sm));                                                                 \
        mlp_simt_kernel<TM_, SAVE_><<<(unsigned)(n_tiles128 * MULT_), 256, sm, st>>>(a);                             \
    } while (0)
    if (nd.L <= 256) {
        if (a.tape) MN_SIMT_LAUNCH(64, true, 2); else MN_SIMT_LAUNCH(64, false, 2);
    } else {
        if (a.tape) MN_SIMT_LAUNCH(32, true, 4); else MN_SIMT_LAUNCH(32, false, 4);
    }
#undef MN_SIMT_LAUNCH
    mn_prof_end(ctx, st);
    MN_LAUNCH_CHECK(ctx);
    return MN_OK;
}
