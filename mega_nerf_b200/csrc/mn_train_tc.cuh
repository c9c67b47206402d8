// Tensor-core training path (precision 'tc_f16' for the recording forward and the backward pass), included inside
// mn_mlp_tc.cu's anonymous namespace.  SURVEY.md §8f-1; the reference trains exactly this way on a GPU: Linear layers in
// fp16 with fp32 accumulation under autocast, gradients scaled into fp16 range (runner.py:243-274, opts.py:99).
//
//   forward   tc_mlp_wg_kernel<PP_TRAIN_FWD>  the inference kernel + every layer's fp16 activations written to a tape in the
//                                             tile-image layout of the activation buffer ([cols/8][128 slots][8]).
//   dgrad     tc_mlp_wg_kernel<PP_DGRAD>      the same GEMM pipeline on transposed weight images: head stage on CUDA cores
//                                             (sigmoid' for a colour head, raw SH coefficients pass through / softplus' /
//                                             rgb Linear transposed), then dH_{l-1} = dZ_l W_l with the
//                                             ReLU mask read from the activation tape in the epilogue; dZ images (fp16, scaled by
//                                             a power of two S) go to a gradient tape.
//   wgrad     tc_wgrad_kernel                 dW_l = dZ_l^T X_l over all slots of a sub-module: both tapes are consumed AS THEY
//                                             ARE through MN-major wgmma descriptors (the slot axis is the K axis; LBO = 128 B
//                                             between 8-slot groups, SBO = 2048 B between 8-column groups), M = 128 output
//                                             channels per CTA (64 per consumer warpgroup), N <= 256 input channels + a 16-column
//                                             all-ones operand whose product is the bias gradient, accumulated in registers over
//                                             a chunk of tiles and flushed with fp32 atomics.  A launch takes a list of Linears
//                                             (WgLinear) and decodes its work item (Linear, output half, X chunk) from blockIdx.y:
//                                             at 256 the fused engine covers every Linear but rgb in one launch; at 512 it makes
//                                             one launch per Linear, and the layer engine one per Linear and tile group.
//   heads     tc_heads_wgrad_kernel (sigma / rgb Linears: 1 and rgb_dim output channels - CUDA cores), tc_emb_grad_kernel
//             (appearance embedding: W_e^T times the per-image sums of dZ_dira rows collected by the dgrad head stage).
//
// Host side (mn_mlp_tc.cu): build_dgrad_plan (the data-gradient chain and the layout of the transposed images,
// packed by tc_dgrad_ready / tc_pack_dgrad), mn_mlp_tc_launch_record and mn_train_tc_backward, shared with the layer-GEMM engine.
#pragma once

// max |g| over the upstream gradient, spread over the machine (an SH head's grad_out has 28 columns per row): every block
// folds a grid-stride share and publishes its maximum with an integer atomicMax on *maxbits (zeroed by the caller; the bit
// patterns of non-negative floats order like the values, and fmaxf drops NaNs, so the result is max |g| exactly).  Only the
// live.rows(rows) rows that hold data are read.
__global__ void tc_grad_absmax_kernel(const float* __restrict__ g, LiveRows live, int64_t rows, int cols, unsigned* __restrict__ maxbits) {
    __shared__ float red[32];
    const int64_t n = live.rows(rows) * cols;
    float m = 0.0f;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) m = fmaxf(m, fabsf(g[i]));
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int i = 1; i < (int)(blockDim.x >> 5); ++i) m = fmaxf(m, red[i]);
        atomicMax(maxbits, __float_as_uint(m));
    }
}
// S = 2^(10 - ceil(log2(max |g|)))  (1 if g == 0 or not finite): the gradient images hold S * dZ in fp16
__global__ void tc_grad_scale_kernel(const unsigned* __restrict__ maxbits, float* __restrict__ scale) {
    if (threadIdx.x == 0) {
        const float m = __uint_as_float(*maxbits);
        float s = 1.0f;
        if (m > 0.0f && m < 3.0e38f) s = exp2f(10.0f - ceilf(log2f(m)));
        scale[0] = fminf(fmaxf(s, 1.0f / 1099511627776.0f), 1099511627776.0f);       // 2^-40 .. 2^40
    }
}

// ------------------------------------------------------------------------------------------------
// weight gradients
// ------------------------------------------------------------------------------------------------
struct WgItem {
    int dz_off;       // byte offset of the 128-column dZ half inside a tile's gradient images
    int x_region;     // 0: activation record, 1: encoder (feature) tile
    int x_off;        // byte offset of the first X column group inside that record
    int n;            // MMA N = X columns (multiple of 16, <= 256)
    int n_real;       // columns that exist in the weight matrix
    int m_real;       // output channels that exist from out0 on (fewer than 128 in a padded last block)
    int w_off;        // float offset of W[out0][in0] inside one sub-module's gradient block
    int k_in;         // row stride (in_features) of that weight matrix
    int b_off;        // float offset of bias[out0], or -1 when another item of the same layer owns the bias
};
// One Linear of a launch: its work items are (128-channel output half, X chunk of <= 256 columns of an input segment)
struct WgLinear {
    WgItem seg[2];                  // input segment s for output channels 0..127 and the segment's first X chunk
    int n_chunks[2];                // X chunks of each input segment (0: no second segment)
    int n_items;                    // (out / 128) * (n_chunks[0] + n_chunks[1])
};
struct WgArgs {
    WgLinear lin[MN_MAX_LAYERS + 2];  // Linears of the launch (trunk, xyz_encoding_final, dir_a_encoding; never rgb), in order
    const unsigned char* act;       // activation records
    const unsigned char* dz;        // gradient images of tile t_min onwards, dz_tile_bytes apart
    const unsigned char* xreg;      // encoder tiles
    int64_t act_tile_bytes, x_tile_bytes, dz_tile_bytes;
    int64_t t_min, t_max;           // tiles covered by the launch
    const int* counters;            // routing counters saved by the forward pass, or NULL (all tiles belong to fixed_sub)
    int fixed_sub;
    LiveRows live;                  // counters == NULL: tiles at or past live.rows(rows) rows hold no tape
    int64_t rows;
    int chunk_tiles;
    float* gw;                      // [n_sub][sub_stride] fp32
    int64_t sub_stride;
    const float* scale;
};
// Last tile + 1 of an unrouted call whose first live.rows(rows) rows hold data.
__device__ __forceinline__ int64_t tc_live_tiles(LiveRows live, int64_t rows) { return (live.rows(rows) + kTileM - 1) / kTileM; }
constexpr int kWgStageBytes = 96 * 1024;
constexpr int kWgThreads = 384;     // warpgroup 0: producer thread; warpgroups 1-2: output channels 0-63 / 64-127 of the item

// Work item y of a launch: the Linear whose items span y, then output channels [128 mh, +128) x input columns [256 c, +256)
// of its segment s.
__device__ __forceinline__ WgItem wg_work_item(const WgArgs& A, int y) {
    int li = 0;
    while (y >= A.lin[li].n_items) y -= A.lin[li++].n_items;
    const WgLinear& l = A.lin[li];
    const int per = l.n_chunks[0] + l.n_chunks[1];
    const int mh = y / per;
    int c = y - mh * per;
    const int s = c < l.n_chunks[0] ? 0 : 1;
    if (s) c -= l.n_chunks[0];
    WgItem it = l.seg[s];
    it.dz_off += mh * 16 * (kTileM * 16);
    it.x_off += c * 32 * (kTileM * 16);
    it.n = min(256, it.n - 256 * c);
    it.n_real = min(256, it.n_real - 256 * c);
    it.m_real -= mh * 128;
    it.w_off += mh * 128 * it.k_in + 256 * c;
    it.b_off = (it.b_off >= 0 && c == 0) ? it.b_off + mh * 128 : -1;
    return it;
}

__global__ void __launch_bounds__(kWgThreads, 1) tc_wgrad_kernel(const WgArgs A) {
    extern __shared__ __align__(1024) unsigned char smem[];
    unsigned char* ring = smem;                                   // 2 x 96 KiB: [dZ half 32 KiB][X <= 64 KiB]
    unsigned char* ones = smem + 2 * kWgStageBytes;               // 6 KiB of fp16 1.0
    uint64_t* bars = reinterpret_cast<uint64_t*>(ones + 6144);
    uint64_t* full = bars;        // [2]
    uint64_t* empty = bars + 2;   // [2], one arrival per consumer warpgroup
    const WgItem it = wg_work_item(A, blockIdx.y);
    int sub = A.fixed_sub;
    int64_t t_lo = A.t_min, t_hi = A.t_max;
    if (A.counters) {
        sub = (int)blockIdx.z;
        t_lo = max(t_lo, (int64_t)(A.counters[CNT_START + sub] / kTileM));
        t_hi = min(t_hi, (int64_t)(A.counters[CNT_START + sub + 1] / kTileM));
    } else {
        t_hi = min(t_hi, tc_live_tiles(A.live, A.rows));
    }
    const int64_t t_begin = t_lo + (int64_t)blockIdx.x * A.chunk_tiles;
    const int64_t t_end = min(t_hi, t_begin + (int64_t)A.chunk_tiles);
    if (t_begin >= t_end) return;

    for (int i = threadIdx.x; i < 6144 / 4; i += kWgThreads) reinterpret_cast<uint32_t*>(ones)[i] = 0x3C003C00u;
    if (threadIdx.x == 0) {
        for (int i = 0; i < 2; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 2); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    fence_proxy_async();
    __syncthreads();
    const uint32_t xbytes = (uint32_t)(it.n / 8) * (kTileM * 16);

    const int wgi = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 7), 0);     // warp-uniform role
    if (wgi == 0) {
        if (threadIdx.x == 0) {
            uint32_t st = 0, ph = 0;
            const unsigned char* xbase = it.x_region ? A.xreg : A.act;
            const int64_t xstride = it.x_region ? A.x_tile_bytes : A.act_tile_bytes;
            for (int64_t t = t_begin; t < t_end; ++t) {
                mbar_wait(&empty[st], ph ^ 1);
                mbar_expect_tx(&full[st], 32768u + xbytes);
                bulk_g2s(ring + (size_t)st * kWgStageBytes, A.dz + (size_t)(t - A.t_min) * A.dz_tile_bytes + it.dz_off, 32768u, &full[st]);
                bulk_g2s(ring + (size_t)st * kWgStageBytes + 32768, xbase + (size_t)t * xstride + it.x_off, xbytes, &full[st]);
                if (++st == 2) { st = 0; ph ^= 1; }
            }
        }
    } else {
        // A = dZ^T (M = 64 channels of this warpgroup x K = 16 slots), B = X^T: both MN-major views of the tile images
        // ([cols/8][128 slots][8]): leading byte offset 128 (next 8 slots), stride byte offset 2048 (next 8 columns).  The
        // all-ones operand turns the bias gradient into one more N = 16 MMA.
        const int wg = wgi - 1;
        const int tid = threadIdx.x & 127, w = tid >> 5, lane = tid & 31, q4 = lane & 3;
        const int ca = 64 * wg + 16 * w + (lane >> 2), cb = ca + 8;      // output channels of this thread's accumulator rows
        const uint64_t od = wg_desc(smem_u32(ones), 128, 2048);
        auto run = [&](auto nm_tag) {
            constexpr int NM = decltype(nm_tag)::value;
            float acc[NM / 2], accb[8];
#pragma unroll
            for (int i = 0; i < NM / 2; ++i) acc[i] = 0.0f;
#pragma unroll
            for (int i = 0; i < 8; ++i) accb[i] = 0.0f;
            wg_fence_operand<NM / 2>(acc);
            wg_fence_operand<8>(accb);
            uint32_t st = 0, ph = 0;
            int prev = -1;
            for (int64_t t = t_begin; t < t_end; ++t) {
                mbar_wait(&full[st], ph);
                const uint32_t base = smem_u32(ring) + st * (uint32_t)kWgStageBytes;
                wg_fence();
#pragma unroll
                for (int ks = 0; ks < 8; ++ks) {
                    const uint64_t ad = wg_desc(base + (uint32_t)ks * 256u + (uint32_t)wg * 16384u, 128, 2048);
                    const uint64_t bd = wg_desc(base + 32768u + (uint32_t)ks * 256u, 128, 2048);
                    wg_mma<NM, 1, 1>(acc, ad, bd, 1u);
                    if (it.b_off >= 0) wg_mma<16, 1, 1>(accb, ad, od, 1u);
                }
                wg_commit();
                if (prev >= 0) {
                    wg_wait<1>();
                    if (tid == 0) mbar_arrive(&empty[prev]);
                }
                prev = (int)st;
                if (++st == 2) { st = 0; ph ^= 1; }
            }
            wg_wait<0>();
            wg_fence_operand<NM / 2>(acc);
            wg_fence_operand<8>(accb);
            // ---- flush: unscale and accumulate into the fp32 gradient block ([out][in] rows of the nn.Linear weight)
            const float inv = 1.0f / *A.scale;
            float* W = A.gw + (size_t)sub * A.sub_stride;
            const bool va = ca < it.m_real, vb = cb < it.m_real;
#pragma unroll
            for (int j = 0; j < NM / 8; ++j) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int c = 8 * j + 2 * q4 + e;
                    if (c < it.n_real) {
                        if (va) atomicAdd(W + it.w_off + (size_t)ca * it.k_in + c, acc[4 * j + e] * inv);
                        if (vb) atomicAdd(W + it.w_off + (size_t)cb * it.k_in + c, acc[4 * j + 2 + e] * inv);
                    }
                }
            }
            if (it.b_off >= 0 && q4 == 0) {
                if (va) atomicAdd(W + it.b_off + ca, accb[0] * inv);
                if (vb) atomicAdd(W + it.b_off + cb, accb[2] * inv);
            }
        };
        if (it.n > 128) run(std::integral_constant<int, 256>{});
        else if (it.n > 64) run(std::integral_constant<int, 128>{});
        else if (it.n > 32) run(std::integral_constant<int, 64>{});
        else run(std::integral_constant<int, 32>{});
    }
}

// sigma Linear (1 x L) and rgb Linear (rgb_dim x L/2) weight / bias gradients from the fp32 head gradients and the fp16 tapes.
struct HeadsArgs {
    const unsigned char* act;
    const float* gf32;              // head-gradient blocks [n_tiles][mn_tc_g32_rows(rgb_dim)][128], of tile t_min onwards
    int64_t act_tile_bytes;
    int L, layers, rgb_dim;
    int cols;                       // columns of an H image in the activation record (L, or padded on the layer engine)
    const int* counters;
    int64_t n_tiles;
    int64_t t_min, t_max;           // tiles covered by gf32 (the layer-GEMM path's tile group; 0 .. n_tiles otherwise)
    LiveRows live;                  // counters == NULL: tiles at or past live.rows(rows) rows hold no tape
    int64_t rows;
    int fixed_sub, chunk_tiles;
    float* gw;
    int64_t sub_stride;
    int sigma_w, sigma_b, rgb_w, rgb_b;     // float offsets in a sub-module's gradient block (rgb_w is [rgb_dim][L/2])
};
// kRgb: 3 for the colour head (exactly 3 rgb rows), MN_TC_RGB_MAX or MN_TC_LG_RGB_MAX for a raw SH head (rgb_dim <= kRgb
// rows).  The rgb weight gradient is split over the channel index k: k accumulates input channel k % (L/2) for the output rows
// [kPer * (k / (L/2)), +kPer) (up to 32 rows: two groups of kPer rows over k < L; up to 80: five groups over k < 5 L/2).  Block z
// of the grid takes the 256 channels k = 256 z + threadIdx.x, so the grid runs max(L, groups x L/2) / 256 channel blocks.
template <int kRgb>
__global__ void __launch_bounds__(256) tc_heads_wgrad_kernel(const HeadsArgs A) {
    constexpr int kPer = kRgb < 16 ? kRgb : 16;       // rgb accumulators per thread
    static_assert(kRgb <= MN_TC_LG_RGB_MAX, "rgb rows of tc_heads_wgrad_kernel (the shared block below, the bias rows k < 1 + kRgb)");
    __shared__ float G[1 + kRgb][kTileM];              // this tile's head-gradient block
    int sub = A.fixed_sub;
    int64_t t_lo = A.t_min, t_hi = min(A.n_tiles, A.t_max);
    if (A.counters) {
        sub = (int)blockIdx.y;
        t_lo = max(t_lo, (int64_t)(A.counters[CNT_START + sub] / kTileM));
        t_hi = min(A.t_max, (int64_t)(A.counters[CNT_START + sub + 1] / kTileM));
    } else {
        t_hi = min(t_hi, tc_live_tiles(A.live, A.rows));
    }
    const int64_t t_begin = t_lo + (int64_t)blockIdx.x * A.chunk_tiles;
    const int64_t t_end = min(t_hi, t_begin + (int64_t)A.chunk_tiles);
    if (t_begin >= t_end) return;
    const int rgb_dim = kRgb == 3 ? 3 : A.rgb_dim;
    const int k = threadIdx.x + 256 * (int)blockIdx.z, L = A.L, half = L / 2, rows = mn_tc_g32_rows(rgb_dim);
    const int kc = k % half, c0 = kPer * (k / half);       // rgb part: input channel, first output row
    const int nc = min(kPer, rgb_dim - c0);                // output rows of this thread (<= 0: none)
    float ws = 0.0f, bs = 0.0f, wr[kPer];
#pragma unroll
    for (int c = 0; c < kPer; ++c) wr[c] = 0.0f;
    for (int64_t t = t_begin; t < t_end; ++t) {
        __syncthreads();
        for (int i = threadIdx.x; i < rows * kTileM; i += 256) G[i / kTileM][i % kTileM] = A.gf32[(size_t)(t - A.t_min) * rows * kTileM + i];
        __syncthreads();
        const unsigned char* rec = A.act + (size_t)t * A.act_tile_bytes;
        if (k < L) {
            const __half* h = reinterpret_cast<const __half*>(rec + mn_tc_img_off(A.layers - 1, A.cols)) + (size_t)(k >> 3) * (kTileM * 8) + (k & 7);
            for (int r = 0; r < kTileM; ++r) ws = fmaf(G[MN_TC_G32_SIGMA][r], __half2float(h[r * 8]), ws);
        }
        if (nc > 0) {
            const __half* g = reinterpret_cast<const __half*>(rec + mn_tc_img_off(A.layers + 1, A.cols)) + (size_t)(kc >> 3) * (kTileM * 8) + (kc & 7);
            for (int r = 0; r < kTileM; ++r) {
                const float gv = __half2float(g[r * 8]);
#pragma unroll
                for (int c = 0; c < kPer; ++c)
                    if (kRgb == 3 || c < nc) wr[c] = fmaf(G[MN_TC_G32_RGB + c0 + c][r], gv, wr[c]);     // colour head: nc == 3
            }
        }
        if (k < rows) for (int r = 0; r < kTileM; ++r) bs += G[k][r];
    }
    float* W = A.gw + (size_t)sub * A.sub_stride;
    if (k < L) atomicAdd(W + A.sigma_w + k, ws);
#pragma unroll
    for (int c = 0; c < kPer; ++c)
        if (c < nc) atomicAdd(W + A.rgb_w + (c0 + c) * half + kc, wr[c]);
    if (k == 0) atomicAdd(W + A.sigma_b, bs);
    else if (k < rows) atomicAdd(W + A.rgb_b + (k - 1), bs);
}

// embedding_a.weight[id][j] += sum_k We[k][j] * S[sub][id][k]     (We = dir_a_encoding columns of the embedding, [L/2][app];
// S rows emb_k >= L/2 floats apart)
__global__ void tc_emb_grad_kernel(const float* __restrict__ emb_sum, int emb_k, const float* __restrict__ packed_bwd, int64_t bwd_stride,
                                   int dira_e, int half, int app, int app_count, float* gw, int64_t sub_stride, int emb_off) {
    const int id = blockIdx.x, sub = blockIdx.y, j = threadIdx.x;
    if (j >= app) return;
    const float* S = emb_sum + ((size_t)sub * app_count + id) * emb_k;
    const float* We = packed_bwd + (size_t)sub * bwd_stride + dira_e;
    float acc = 0.0f;
    bool any = false;
    for (int k = 0; k < half; ++k) {
        const float s = S[k];
        any |= s != 0.0f;
        acc = fmaf(We[k * app + j], s, acc);
    }
    if (any) atomicAdd(gw + (size_t)sub * sub_stride + emb_off + (size_t)id * app + j, acc);
}
