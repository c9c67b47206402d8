#pragma once

// Layer-GEMM path for every network the fused kernel does not take: layer_dim 64..4096 of any value, 1..MN_MAX_LAYERS trunk
// layers, and the spherical-harmonics heads of degree 3 and 4 (32 < rgb_dim <= MN_TC_LG_RGB_MAX) at every width.  Its rgb head
// is not a GEMM, so a wider head needs no new tiling.  N is padded to 256-column blocks and every activation image to a multiple
// of 128 columns (lg_cols in mn_mlp_tc.cu), with zero weights and biases in the padding: the padded columns are exactly 0, and
// each GEMM reads its input images' padded width as K, so no kernel here has an N or K tail.  Included inside mn_mlp_tc.cu's
// anonymous namespace after mn_mlp_wg.cuh (whose wgmma wrappers it uses).
//
// One 128-row tile of 2048-wide fp16 activations is 512 KiB and one 2048 x 2048 layer 8 MiB of fp16 weights, so neither
// fits in shared memory.  Each Linear of the network is one launch of tc_layer_gemm_kernel, Y = act(X W^T + b), with the
// activations of a tile group in HBM between launches.  At 2048 columns a row reads 4 KiB and writes 4 KiB per layer for
// 8.4 MFLOP, about 1000 FLOP per HBM byte, so the GEMMs stay bound by the tensor cores.
//
//   tc_layer_gemm_kernel<kSplit>   persistent, 384 threads; work item = (128-slot tile, 256-column N block).  The N blocks
//                                  of one tile are adjacent in the schedule, so the tile's A operand is read from HBM about
//                                  once and from L2 for the other N blocks.
//     warpgroup 2     one thread streams K-slabs of A (the tile image, [K/8][128][8]) and of B (the N block of the weight
//                     image, [N/256][K/8][256][8]) with 1-D cp.async.bulk copies into an mbarrier ring
//     warpgroups 0-1  rows 0-63 / 64-127: wgmma m64n256k16, fp32 accumulators in registers that start at the bias;
//                     epilogue straight from the registers: ReLU (none for xyz_encoding_final), fp16, stored to the output
//                     tile image in HBM (a quad of lanes writes one row's 16 bytes).
//     kSplit (tc_f16x3): each stage carries hi and lo planes of both operands; three MMAs per K step (hi*hi + hi*lo + lo*hi),
//     and the epilogue stores the fp16 residual of every activation in the output's lo plane.
//   tc_layer_head_kernel   one thread per tile row, CUDA cores, fp32: sigma = the last trunk activations . sigma_w + bias
//                          (+ sigma_noise) -> ReLU / shifted softplus; rgb = W_rgb G (or W_rgb H_last without dir_a_encoding)
//                          -> tc_emit_rgb.  sigma_only stops after sigma.  A recording (training) call also fills the tile's
//                          fp32 head block of the tensor-core tape.  <32> for rgb_dim <= 32, <MN_TC_LG_RGB_MAX> above: the
//                          rgb accumulators of a row stay in registers either way.
//
// Training (precision tc_f16, mn_train_tc.cuh): the recording forward is the same launch list with the encoder tiles and every
// GEMM's output written to the tape instead of the group buffers.  The backward runs the data-gradient chain through
// tc_layer_gemm_kernel<false, true>: A = the scaled fp16 gradient image of a Linear's output, B = a transposed weight image
// ([in/256][out/8][256][8]), and an epilogue that adds S dsigma x sigma_w (last trunk layer) and applies the ReLU mask read
// from the activation tape at the (row, column) it stores.  tc_layer_head_dgrad_kernel is its head stage.
//
// A Linear has one or two K segments: the tile's encoder features (kpe or kaux columns of the feature tile image) and / or
// the previous activations (an activation buffer of the group).  Skip layers read [PE, H], dir_a_encoding reads [F, aux].
// The host side is in mn_mlp_tc.cu: build_plan maps the Linear table (tc_linears) to the forward GEMMs of either engine,
// lg_net derives this engine's activation buffers and rgb head from that plan, and lg_gemm launches one GEMM of the forward
// (layer_launch) or of the backward's data-gradient chain (mn_train_tc_backward, images in build_dgrad_plan's layout).

constexpr int kLgGroupTiles = 384;       // tiles per group: bounds the activation workspace (see mn_mlp_tc_workspace)
constexpr int kLgStages = 4;             // ring stages of 48 KiB
constexpr int kLgBlock = 256;            // N columns of one work item

struct LgArgs {
    MlpArgs m;                           // routing: sub-module of a tile, device-side slot count
    int64_t tile0;                       // first (global) tile of the group
    int64_t n_tiles;                     // tiles of the group
    const unsigned char* wpack;          // per sub-module: [hi plane][lo plane][fp32 block]
    int64_t sub_bytes, w_lo;             // bytes per sub-module; offset of the lo plane
    int w_off, k_tot, n_blk, n_out, bias_off, f32_off, relu;
    int nseg;
    const unsigned char* a[2];           // A segments: tile 0 of the group (hi plane)
    int ak[2];                           // K columns of each segment (multiple of 16)
    int64_t a_tile_bytes[2], a_lo[2];    // tile stride and lo-plane offset of each segment's source
    unsigned char* out;                  // output image of tile 0 of the group, [n_blk * 256 / 8][128][8]
    int64_t out_tile_bytes, out_lo;
    // kDgrad: no bias.  mask: activation image of the output (tile 0 of the group), NULL for xyz_encoding_final (no
    // activation).  dsig: d sigma pre-activation per slot (unscaled fp32, tile stride dsig_tile_floats), NULL except for the
    // last trunk layer, whose sigma weights sit in the fp32 block at bias_off.  scale: the gradient scale S.
    const unsigned char* mask;
    int64_t mask_tile_bytes;
    const float* dsig;
    int64_t dsig_tile_floats;
    const float* scale;
};

template <bool kSplit>
struct LgShape {
    static constexpr int slab = kSplit ? 32 : 64;                    // K columns per stage
    static constexpr int a_bytes = slab * kTileM * 2;                // 16 / 8 KiB
    static constexpr int b_bytes = slab * kLgBlock * 2;              // 32 / 16 KiB
    static constexpr int planes = kSplit ? 2 : 1;
    static constexpr int stage_bytes = (a_bytes + b_bytes) * planes; // [A hi][A lo][B hi][B lo]: 48 KiB
    static constexpr int smem = kLgStages * stage_bytes + 256;
};

// The K-slab walk of one work item, shared by the producer and the consumers: f(kc, a_src, b_src) per ring stage.
template <class F>
__device__ __forceinline__ void lg_walk(const LgArgs& A, int64_t lt, const unsigned char* wblk, int slab, F&& f) {
    int kbase = 0;
    for (int s = 0; s < A.nseg; ++s) {
        const unsigned char* asrc = A.a[s] + lt * A.a_tile_bytes[s];
        const int ks = A.ak[s];
        for (int k0 = 0; k0 < ks; k0 += slab) {
            const int kc = ks - k0 < slab ? ks - k0 : slab;
            f(kc, s, asrc + (size_t)k0 * (kTileM * 2), wblk + (size_t)(kbase + k0) * (kLgBlock * 2));
        }
        kbase += ks;
    }
}

template <bool kSplit, bool kDgrad = false>
__global__ void __launch_bounds__(kWgmmaThreads, 1) tc_layer_gemm_kernel(const LgArgs A) {
    extern __shared__ __align__(1024) unsigned char smem[];
    using S = LgShape<kSplit>;
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + kLgStages * S::stage_bytes);
    uint64_t* empty = full + kLgStages;          // one arrival per consumer warpgroup

    const int64_t n_slots = A.m.n_slots();
    int64_t n_tiles = (n_slots + kTileM - 1) / kTileM - A.tile0;     // tiles at or past n_slots exit early
    if (n_tiles > A.n_tiles) n_tiles = A.n_tiles;
    const int64_t n_items = n_tiles > 0 ? n_tiles * A.n_blk : 0;

    if (threadIdx.x == 0) {
        for (int i = 0; i < kLgStages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 2); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    const int wgi = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 7), 0);
    if (wgi == 2) {
        // =========================== producer ===========================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kWgProducerRegs));
        if (threadIdx.x == 256) {
            int stage = 0;
            uint32_t phase = 0;
            for (int64_t it = blockIdx.x; it < n_items; it += gridDim.x) {
                const int64_t lt = it / A.n_blk;
                const int nb = (int)(it - lt * A.n_blk);
                const unsigned char* wblk = A.wpack + (size_t)A.m.sub_of_tile(A.tile0 + lt) * A.sub_bytes + A.w_off +
                                            (size_t)nb * A.k_tot * (kLgBlock * 2);
                lg_walk(A, lt, wblk, S::slab, [&](int kc, int s, const unsigned char* asrc, const unsigned char* bsrc) {
                    mbar_wait(&empty[stage], phase ^ 1);
                    const uint32_t ab = (uint32_t)kc * kTileM * 2, bb = (uint32_t)kc * kLgBlock * 2;
                    mbar_expect_tx(&full[stage], (ab + bb) * S::planes);
                    unsigned char* sb = smem + (size_t)stage * S::stage_bytes;
                    bulk_g2s(sb, asrc, ab, &full[stage]);
                    bulk_g2s(sb + S::planes * S::a_bytes, bsrc, bb, &full[stage]);
                    if (kSplit) {
                        bulk_g2s(sb + S::a_bytes, asrc + A.a_lo[s], ab, &full[stage]);
                        bulk_g2s(sb + 2 * S::a_bytes + S::b_bytes, bsrc + A.w_lo, bb, &full[stage]);
                    }
                    if (++stage == kLgStages) { stage = 0; phase ^= 1; }
                });
            }
        }
    } else {
        // =========================== consumers: MMA + epilogue ===========================
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kWgConsumerRegs));
        const int wg = wgi;
        const int t = threadIdx.x & 127, w = t >> 5, lane = t & 31, q4 = lane & 3;
        // accumulator fragment of m64n256k16: rows ra, ra + 8; in column group j, columns 8j + 2 q4 + {0, 1}
        const int ra = 64 * wg + 16 * w + (lane >> 2);
        const uint32_t smem_s = smem_u32(smem);
        const uint32_t row_base = (uint32_t)(64 * wg * 16);
        int stage = 0;
        uint32_t phase = 0;
        for (int64_t it = blockIdx.x; it < n_items; it += gridDim.x) {
            const int64_t lt = it / A.n_blk;
            const int nb = (int)(it - lt * A.n_blk);
            const int sub = A.m.sub_of_tile(A.tile0 + lt);
            // kDgrad: sigma weights (last trunk layer) or nothing at bias_off
            const float* bias = reinterpret_cast<const float*>(A.wpack + (size_t)sub * A.sub_bytes + A.f32_off) + A.bias_off + nb * kLgBlock;
            // the forward's accumulators start at the bias (wgmma computes D = A B + D), so its epilogue has no bias to add;
            // rows ra and ra + 8 take column c's bias: acc[4 j .. 4 j + 3] = (ra, c), (ra, c + 1), (ra + 8, c), (ra + 8, c + 1)
            float acc[128];
#pragma unroll
            for (int j = 0; j < 32; ++j) {
                const float2 bv = kDgrad ? make_float2(0.0f, 0.0f) : __ldg(reinterpret_cast<const float2*>(bias + 8 * j + 2 * q4));
                acc[4 * j] = bv.x; acc[4 * j + 1] = bv.y; acc[4 * j + 2] = bv.x; acc[4 * j + 3] = bv.y;
            }
            wg_fence_operand<128>(acc);
            int prev = -1;
            uint32_t accum = kDgrad ? 0u : 1u;
            lg_walk(A, lt, nullptr, S::slab, [&](int kc, int, const unsigned char*, const unsigned char*) {
                mbar_wait(&full[stage], phase);
                const uint32_t sa = smem_s + (uint32_t)(stage * S::stage_bytes);
                const uint32_t sbb = sa + S::planes * S::a_bytes;
                wg_fence();
                for (int kk = 0; kk < kc; kk += 16) {
                    const uint64_t ad = wg_desc(sa + (uint32_t)(kk >> 3) * (kTileM * 16) + row_base, kTileM * 16, 128);
                    const uint64_t bd = wg_desc(sbb + (uint32_t)(kk >> 3) * (kLgBlock * 16), kLgBlock * 16, 128);
                    wg_mma<256>(acc, ad, bd, accum);
                    accum = 1;
                    if (kSplit) {
                        const uint64_t adl = wg_desc(sa + S::a_bytes + (uint32_t)(kk >> 3) * (kTileM * 16) + row_base, kTileM * 16, 128);
                        const uint64_t bdl = wg_desc(sbb + S::b_bytes + (uint32_t)(kk >> 3) * (kLgBlock * 16), kLgBlock * 16, 128);
                        wg_mma<256>(acc, ad, bdl, 1);
                        wg_mma<256>(acc, adl, bd, 1);
                    }
                }
                wg_commit();
                // the MMAs of the previous stage have completed: release it (one arrival per warpgroup)
                if (prev >= 0) {
                    wg_wait<1>();
                    if (t == 0) mbar_arrive(&empty[prev]);
                }
                prev = stage;
                if (++stage == kLgStages) { stage = 0; phase ^= 1; }
            });
            wg_wait<0>();
            wg_fence_operand<128>(acc);
            if (prev >= 0 && t == 0) mbar_arrive(&empty[prev]);

            // epilogue: activation, fp16 [+ residual] -> output tile image in HBM
            const size_t po = (size_t)nb * (kLgBlock / 8) * (kTileM * 16) + (size_t)ra * 16 + q4 * 4;
            unsigned char* o = A.out + lt * A.out_tile_bytes + po;
            if constexpr (kDgrad) {
                // data gradient: the accumulators hold S dH; [+ S dsigma x sigma_w]; dZ = dH where the activation is > 0
                const unsigned char* mk = A.mask ? A.mask + lt * A.mask_tile_bytes + po : nullptr;
                float dsa = 0.0f, dsb = 0.0f;
                if (A.dsig) {
                    const float S = *A.scale;
                    dsa = A.dsig[lt * A.dsig_tile_floats + ra] * S;
                    dsb = A.dsig[lt * A.dsig_tile_floats + ra + 8] * S;
                }
                // the mask and sigma-weight loads of JB column groups are issued together
                constexpr int JB = 8;
#pragma unroll
                for (int j0 = 0; j0 < 32; j0 += JB) {
                    __half2 ma[JB], mb[JB];
                    float2 sv[JB];
#pragma unroll
                    for (int jj = 0; jj < JB; ++jj) {
                        const int j = j0 + jj;
                        ma[jj] = mb[jj] = __float2half2_rn(1.0f);
                        sv[jj] = make_float2(0.0f, 0.0f);
                        if (nb * kLgBlock + 8 * j >= A.n_out) continue;
                        if (mk) {
                            ma[jj] = *reinterpret_cast<const __half2*>(mk + (size_t)j * (kTileM * 16));
                            mb[jj] = *reinterpret_cast<const __half2*>(mk + (size_t)j * (kTileM * 16) + 128);
                        }
                        if (A.dsig) sv[jj] = __ldg(reinterpret_cast<const float2*>(bias + 8 * j + 2 * q4));
                    }
#pragma unroll
                    for (int jj = 0; jj < JB; ++jj) {
                        const int j = j0 + jj;
                        if (nb * kLgBlock + 8 * j >= A.n_out) continue;
                        float a0 = acc[4 * j], a1 = acc[4 * j + 1], b0 = acc[4 * j + 2], b1 = acc[4 * j + 3];
                        if (A.dsig) {
                            a0 = fmaf(dsa, sv[jj].x, a0); a1 = fmaf(dsa, sv[jj].y, a1);
                            b0 = fmaf(dsb, sv[jj].x, b0); b1 = fmaf(dsb, sv[jj].y, b1);
                        }
                        if (!(__low2float(ma[jj]) > 0.0f)) a0 = 0.0f;
                        if (!(__high2float(ma[jj]) > 0.0f)) a1 = 0.0f;
                        if (!(__low2float(mb[jj]) > 0.0f)) b0 = 0.0f;
                        if (!(__high2float(mb[jj]) > 0.0f)) b1 = 0.0f;
                        unsigned char* p = o + (size_t)j * (kTileM * 16);
                        *reinterpret_cast<uint32_t*>(p) = pack_h2(a0, a1);
                        *reinterpret_cast<uint32_t*>(p + 128) = pack_h2(b0, b1);
                    }
                }
                continue;
            }
#pragma unroll
            for (int j = 0; j < 32; ++j) {
                if (nb * kLgBlock + 8 * j >= A.n_out) continue;
                float a0 = acc[4 * j], a1 = acc[4 * j + 1], b0 = acc[4 * j + 2], b1 = acc[4 * j + 3];
                if (A.relu) { a0 = fmaxf(a0, 0.0f); a1 = fmaxf(a1, 0.0f); b0 = fmaxf(b0, 0.0f); b1 = fmaxf(b1, 0.0f); }
                const uint32_t ha = pack_h2(a0, a1), hb = pack_h2(b0, b1);
                unsigned char* p = o + (size_t)j * (kTileM * 16);
                *reinterpret_cast<uint32_t*>(p) = ha;
                *reinterpret_cast<uint32_t*>(p + 128) = hb;
                if (kSplit) {
                    const float2 fa = __half22float2(*reinterpret_cast<const __half2*>(&ha));
                    const float2 fb = __half22float2(*reinterpret_cast<const __half2*>(&hb));
                    *reinterpret_cast<uint32_t*>(p + A.out_lo) = pack_h2(a0 - fa.x, a1 - fa.y);
                    *reinterpret_cast<uint32_t*>(p + A.out_lo + 128) = pack_h2(b0 - fb.x, b1 - fb.y);
                }
            }
        }
    }
    __syncthreads();
}

struct LhArgs {
    MlpArgs m;
    int64_t tile0;
    const unsigned char* wpack;
    int64_t sub_bytes;
    int f32_off, sigma_w_off, rgb_w_off, rgb_b_off;   // fp32 block: byte offset; float offsets inside it
    const unsigned char* h;                           // last trunk activations of tile 0 of the group, [L/8][128][8]
    int64_t h_tile_bytes, h_lo;                       // lo-plane offset (tc_f16x3) or 0
    const unsigned char* g;                           // rgb head input: G, or the last trunk activations
    int64_t g_tile_bytes, g_lo;
    int L, rgb_in;                                    // columns the sigma / rgb loops read: L, rgb_in rounded up to 8 (zero weights)
    float* tape_f32;                                 // recording call: fp32 head blocks of the tape [tiles][MN_TC_F32_ROWS][128], or NULL
};

// 8 consecutive columns c0 .. c0 + 7 of row t of a tile image, as fp32 (hi + lo when the lo plane exists)
__device__ __forceinline__ void lg_load8(const unsigned char* img, int64_t lo, int c0, int t, float* v) {
    const size_t off = (size_t)(c0 >> 3) * (kTileM * 16) + (size_t)t * 16;
    const uint4 hv = *reinterpret_cast<const uint4*>(img + off);
    const __half2* hh = reinterpret_cast<const __half2*>(&hv);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const float2 f = __half22float2(hh[e]);
        v[2 * e] = f.x;
        v[2 * e + 1] = f.y;
    }
    if (lo) {
        const uint4 lv = *reinterpret_cast<const uint4*>(img + lo + off);
        const __half2* lh = reinterpret_cast<const __half2*>(&lv);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float2 f = __half22float2(lh[e]);
            v[2 * e] += f.x;
            v[2 * e + 1] += f.y;
        }
    }
}

// kR bounds rgb_dim (mn_tc_lg_rgb_bound): 32, or MN_TC_LG_RGB_MAX for the SH heads of degree 3 and 4.
template <int kR>
__global__ void __launch_bounds__(kTileM) tc_layer_head_kernel(const LhArgs A) {
    const int t = threadIdx.x;
    const int64_t tile = A.tile0 + blockIdx.x;
    const int64_t n_slots = A.m.n_slots();
    const int64_t slot = tile * kTileM + t;
    const int64_t row = A.m.row_of_slot(slot, n_slots);
    float* tf = A.tape_f32 ? A.tape_f32 + (size_t)tile * MN_TC_F32_ROWS * kTileM + t : nullptr;
    if (row < 0) {
        if (tf) {       // padding slot: finite values for the backward's head stage (its upstream gradient is zero)
            tf[MN_TC_F32_SIGMA * kTileM] = 0.0f;
            for (int c = 0; c < 3; ++c) tf[(MN_TC_F32_RGB + c) * kTileM] = 0.5f;
            tf[MN_TC_F32_ID * kTileM] = 0.0f;
        }
        return;
    }
    const int sub = A.m.sub_of_tile(tile);
    const float* f32 = reinterpret_cast<const float*>(A.wpack + (size_t)sub * A.sub_bytes + A.f32_off);
    float v[8];

    const float* sw = f32 + A.sigma_w_off;
    const unsigned char* h = A.h + (int64_t)blockIdx.x * A.h_tile_bytes;
    float s = 0.0f;
    for (int c = 0; c < A.L; c += 8) {
        lg_load8(h, A.h_lo, c, t, v);
        const float4 wa = __ldg(reinterpret_cast<const float4*>(sw + c)), wb = __ldg(reinterpret_cast<const float4*>(sw + c + 4));
        s = fmaf(v[0], wa.x, s); s = fmaf(v[1], wa.y, s); s = fmaf(v[2], wa.z, s); s = fmaf(v[3], wa.w, s);
        s = fmaf(v[4], wb.x, s); s = fmaf(v[5], wb.y, s); s = fmaf(v[6], wb.z, s); s = fmaf(v[7], wb.w, s);
    }
    s = s + sw[A.L];                                  // sigma bias is stored right after sigma_w
    if (A.m.sigma_noise) s = s + A.m.sigma_noise[row];
    if (tf) {
        tf[MN_TC_F32_SIGMA * kTileM] = s;                 // pre-activation (with the density noise)
        tf[MN_TC_F32_ID * kTileM] = A.m.nd.app > 0 ? A.m.src.index(row) : 0.0f;
    }
    const float sg = A.m.nd.softplus ? mn_softplus_shifted(s) : fmaxf(s, 0.0f);
    if (A.m.sigma_only) {
        const int64_t o = (A.m.scatter ? row : slot) * A.m.out_cols;
        A.m.out[o] = A.m.slot_w ? sg * A.m.slot_w[slot] : sg;
        return;
    }

    // rgb Linear over the head input, rgb_dim rows of [rgb_dim][rgb_in] fp32 weights.  Only compile-time indices into acc
    // (loops unrolled to kR and left at r == R), so the array stays in registers.
    const int R = A.m.nd.rgb_dim;
    const float* wr = f32 + A.rgb_w_off;
    const unsigned char* g = A.g + (int64_t)blockIdx.x * A.g_tile_bytes;
    float acc[kR];
#pragma unroll
    for (int r = 0; r < kR; ++r) acc[r] = 0.0f;
    for (int c = 0; c < A.rgb_in; c += 8) {
        lg_load8(g, A.g_lo, c, t, v);
#pragma unroll
        for (int r = 0; r < kR; ++r) {
            if (r >= R) break;
            const float4 wa = __ldg(reinterpret_cast<const float4*>(wr + (size_t)r * A.rgb_in + c));
            const float4 wb = __ldg(reinterpret_cast<const float4*>(wr + (size_t)r * A.rgb_in + c + 4));
            float x = acc[r];
            x = fmaf(v[0], wa.x, x); x = fmaf(v[1], wa.y, x); x = fmaf(v[2], wa.z, x); x = fmaf(v[3], wa.w, x);
            x = fmaf(v[4], wb.x, x); x = fmaf(v[5], wb.y, x); x = fmaf(v[6], wb.z, x); x = fmaf(v[7], wb.w, x);
            acc[r] = x;
        }
    }
    uint32_t raw[kR];
#pragma unroll
    for (int r = 0; r < kR; ++r) raw[r] = __float_as_uint(acc[r]);
    tc_emit_rgb<kR>(A.m, sub, row, slot, raw, f32 + A.rgb_b_off, sg, tf ? tf + MN_TC_F32_RGB * kTileM : nullptr);
}

// ---- training backward: head stage of one tile group, one thread per tile row (CUDA cores, fp32).  Upstream gradient x blend
// weight -> sigmoid' (colour head) or the raw SH coefficients / softplus' or ReLU' -> the head-gradient block (unscaled) and
// dZ_G = mask(G > 0) (W_rgb^T d rgb) as a scaled fp16 tile image; per-image sums of dZ_G rows for the appearance embedding.
struct LdArgs {
    MlpArgs m;                                        // routing, blend weights, nd
    int64_t tile0;
    const float* grad_out;                            // [rows][rgb_dim + 1]
    const float* tape_f32;                            // fp32 head blocks of the tape (all tiles)
    const unsigned char* g;                           // G activation image of tile 0 of the group (tape)
    int64_t g_tile_bytes;
    const unsigned char* wpack;                       // forward pack: rgb weights [rgb_dim][rgb_k] in the fp32 block
    int64_t sub_bytes;
    int f32_off, rgb_w_off;
    int rgb_k;                                        // L/2 rounded up to 8: the weight rows' stride, zero past L/2
    int cols;                                         // columns of a dZ_G image (L/2 padded; zeros from rgb_k on)
    float* gf32;                                      // head-gradient blocks of the group [tiles][mn_tc_g32_rows][128]
    unsigned char* dz;                                // dZ_G images of the group [tiles][cols/8][128][8], S x dZ in fp16
    float* emb_sum;                                   // [n_sub][app_count][rgb_k] or NULL
    const float* scale;
};

template <int kR>
__global__ void __launch_bounds__(kTileM) tc_layer_head_dgrad_kernel(const LdArgs A) {
    const int t = threadIdx.x, lane = t & 31;
    const int64_t tile = A.tile0 + blockIdx.x;
    const int64_t n_slots = A.m.n_slots();
    if (tile * kTileM >= n_slots) return;
    const int64_t slot = tile * kTileM + t;
    const int64_t row = A.m.row_of_slot(slot, n_slots);
    const int sub = A.m.sub_of_tile(tile);
    const int R = A.m.nd.rgb_dim, rk = A.rgb_k;
    const float S = *A.scale;
    const float* tf = A.tape_f32 + (size_t)tile * MN_TC_F32_ROWS * kTileM + t;
    float d[kR];
    const float ds = tc_head_grad<kR>(A.m, A.grad_out, row, slot, tf, d);
    float* tg = A.gf32 + (size_t)blockIdx.x * mn_tc_g32_rows(R) * kTileM + t;
    tg[MN_TC_G32_SIGMA * kTileM] = ds;
#pragma unroll
    for (int c = 0; c < kR; ++c) {
        if (c >= R) break;
        tg[(MN_TC_G32_RGB + c) * kTileM] = d[c];
    }
    const int id = (int)tf[MN_TC_F32_ID * kTileM];
    const float* Wr = reinterpret_cast<const float*>(A.wpack + (size_t)sub * A.sub_bytes + A.f32_off) + A.rgb_w_off;
    const unsigned char* gimg = A.g + (int64_t)blockIdx.x * A.g_tile_bytes + (size_t)t * 16;
    unsigned char* dimg = A.dz + (int64_t)blockIdx.x * A.cols * (kTileM * 2) + (size_t)t * 16;
    float* sums = A.emb_sum ? A.emb_sum + (size_t)sub * A.m.nd.app_count * rk : nullptr;
    for (int k0 = 0; k0 < rk; k0 += 8) {
        float v[8];
        tc_rgb_dgrad8<kR>(Wr, rk, k0, d, R, gimg + (size_t)(k0 >> 3) * (kTileM * 16), v);
        if (sums) tc_emb_sums8(sums + k0, rk, row >= 0, id, lane, v);
        uint32_t pk[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) pk[e] = pack_h2(v[2 * e] * S, v[2 * e + 1] * S);
        *reinterpret_cast<uint4*>(dimg + (size_t)(k0 >> 3) * (kTileM * 16)) = make_uint4(pk[0], pk[1], pk[2], pk[3]);
    }
    // the image's padding columns: zero gradients for the data-gradient GEMM and the weight gradient of dir_a_encoding
    for (int k0 = rk; k0 < A.cols; k0 += 8) *reinterpret_cast<uint4*>(dimg + (size_t)(k0 >> 3) * (kTileM * 16)) = make_uint4(0, 0, 0, 0);
}
