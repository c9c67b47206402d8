// MN_PREC_TC_F16 / MN_PREC_TC_F16X3: the NeRF MLP (models/nerf.py:115-160) on the Hopper tensor cores.
//
//   tc_encode_kernel   sample rows -> fp16 feature tiles (positional encodings of xyz / dir, appearance
//                      embedding) written in the exact shared-memory operand image, one 128-row tile
//                      per CTA, coalesced 16-byte stores (tc_encode_fast_kernel: the common shape).
//   tc_mlp_wg_kernel   persistent, warp-specialised (mn_mlp_wg.cuh): one producer thread (cp.async.bulk of
//                      weight K-slabs through an mbarrier ring and of the feature tiles), two consumer
//                      warpgroups issuing wgmma.mma_async (accumulators in registers) and running the
//                      epilogue (bias/ReLU -> fp16 -> next layer's A operand, in registers for tc_f16 inference up to
//                      256 wide and in shared memory otherwise; heads -> HBM).
//                      Activations never leave the SM between layers.
//
// Operand layout (both A tiles and packed weights): K-major, no swizzle, "interleaved" core matrices:
//   element (row r, col k) of an R-row operand lives at byte (k/8)*(R*16) + r*16 + (k%8)*2,
// i.e. [K/8][R][8] fp16.  wgmma descriptor: LBO = R*16 (next 8-column chunk), SBO = 128 (next 8-row group).
// The epilogue's per-row 16-byte stores and the packer's images are contiguous in this layout, any K that
// is a multiple of 16 works, and no TMA tensor map is needed (plain 1-D bulk copies).
//
// Every other network of 64..4096 wide and 1..16 trunk layers, and the spherical-harmonics heads of degree 3 and 4 (rgb_dim 48,
// 75) at any width, run on the layer-GEMM engine instead (mn_layer_gemm.cuh).  Host side: tc_linears lists the
// network's Linears once; tc_net picks the engine and the training coverage from that table, and builds the forward plan of
// either engine (build_plan) and the data-gradient plan (build_dgrad_plan), once per model (mn_model::tc, build_layout).
// mn_mlp_tc_pack writes the forward images of either engine, tc_dgrad_ready / tc_pack_dgrad the transposed images of the
// backward, and mn_train_tc_backward runs the backward of either engine between one shared workspace carve, gradient scale
// and head / embedding epilogue.
#include <cuda_fp16.h>

#include <type_traits>
#include <vector>

#include "mn_model.cuh"

namespace {

constexpr int kTileM = MN_TILE;

// kernel modes of tc_mlp_wg_kernel (the test hook mn_debug_tp_program_mode names them MN_TP_*)
enum { PP_INFER = 0, PP_TRAIN_FWD = 1, PP_DGRAD = 2 };
static_assert(PP_INFER == MN_TP_INFER && PP_TRAIN_FWD == MN_TP_TRAIN_FWD && PP_DGRAD == MN_TP_DGRAD, "mn_debug_tp_program_mode modes");

int pad16(int x) { return (x + 15) / 16 * 16; }
int pad8(int x) { return (x + 7) / 8 * 8; }

// Layer engine: every activation image (and so every hidden K segment) is padded to a multiple of kLgCols columns, the
// 128-channel output block of the weight-gradient kernel.  The padded columns hold exactly 0: zero weights and zero bias,
// then ReLU (or none), so every GEMM reads whole K slabs and no kernel has a column tail.
constexpr int kLgCols = 128;
int lg_cols(int x) { return (x + kLgCols - 1) / kLgCols * kLgCols; }

// layer: the table of the layer engine, whose activation images are padded to lg_cols; the fused engine's are not.
TcLinears tc_linears(const mn_model& m, bool layer) {
    const NetDims& nd = m.nd;
    TcLinears T{};
    T.kpe = pad16(nd.in_xyz);
    T.kaux = nd.aux > 0 ? pad16(nd.aux) : 0;
    T.hc = layer ? lg_cols(nd.L) : nd.L;
    T.gc = layer ? lg_cols(nd.L / 2) : nd.L / 2;
    const TcSeg pe{SRC_XPE, T.kpe, nd.in_xyz, 0};
    const TcSeg hs{SRC_H, T.hc, nd.L, 0};              // the previous Linear's H or F image
    auto add = [&](int n, int cols, TcSeg s0, int kin, int w, int b, int bwd, int epi) -> TcLinear& {
        TcLinear& l = T.l[T.n++];
        l = TcLinear{n, cols, 1, {s0, {}}, kin, w, b, bwd, epi};
        return l;
    };
    for (int i = 0; i < nd.layers; ++i) {
        TcLinear& l = add(nd.L, T.hc, i == 0 ? pe : hs, m.lay.kin[i], m.lay.w[i], m.lay.b[i], i > 0 ? m.blay.w[i] : -1,
                          i == nd.layers - 1 ? EPI_RELU_SIGMA : EPI_RELU);
        if (i > 0 && ((nd.skip_mask >> i) & 1)) {      // cat[PE, h]: PE columns first
            l.nseg = 2;
            l.seg[0] = pe;
            l.seg[1] = TcSeg{SRC_H, T.hc, nd.L, nd.in_xyz};
        }
    }
    T.n_trunk = T.n;
    if (nd.has_dir_a) {                                // has_dir_a implies aux > 0: dir_a_encoding reads [F, dir PE + embedding]
        add(nd.L, T.hc, hs, nd.L, m.lay.final_w, m.lay.final_b, m.blay.final_w, EPI_LINEAR);
        TcLinear& d = add(nd.L / 2, T.gc, hs, nd.L + nd.aux, m.lay.dira_w, m.lay.dira_b, m.blay.dira_f, EPI_RELU);
        d.nseg = 2;
        d.seg[1] = TcSeg{SRC_XAUX, T.kaux, nd.aux, nd.L};
    }
    add(nd.rgb_dim, nd.rgb_dim, TcSeg{SRC_H, nd.rgb_in, nd.rgb_in, 0}, nd.rgb_in, m.lay.rgb_w, m.lay.rgb_b, -1, EPI_RGB);
    return T;
}

// ---- forward plan of either engine: one GEMM per Linear, the weight images back to back in a precision plane, the fp32 block
// [biases][sigma_w (L)][sigma_b (4)].  The fused engine (tc_mlp_wg_kernel) runs every GEMM in one launch, the rgb head as an
// N = 32 GEMM, and reserves bstride floats per bias.  The layer engine (mn_layer_gemm.cuh) launches one GEMM per Linear with
// N padded to 256-column blocks, in the image and in the bias, and K padded as its input images are (TcLinears::hc); its rgb
// head is not a GEMM: tc_layer_head_kernel reads [rgb_w [rgb_dim][pad8(rgb_in)]][rgb_b (mn_tc_lg_rgb_bound(rgb_dim))] from
// the end of the fp32 block (lg_net), and sigma_w takes pad8(L) floats there.  The fp32 padding is zero (the pack is zeroed
// once at allocation and repacks write only the real entries), so the head loops run over whole groups of 8 columns.
void build_plan(const NetDims& nd, const TcLinears& T, bool layer, TcPlan* p) {
    TcPlan& P = *p;
    P = TcPlan{};
    P.L = nd.L;
    P.bstride = layer ? 0 : nd.L > 256 ? 512 : 256;
    P.kpe = T.kpe;
    P.kaux = T.kaux;
    P.n_trunk = T.n_trunk;
    P.n_gemm = layer ? T.n - 1 : T.n;
    int woff = 0, foff = 0;
    for (int gi = 0; gi < P.n_gemm; ++gi) {
        const TcLinear& l = T.l[gi];
        TcGemm& g = P.g[gi];
        g.n = layer ? (l.n + 255) / 256 * 256 : l.epi == EPI_RGB ? 32 : l.n;
        g.nseg = l.nseg;
        for (int s = 0; s < l.nseg; ++s) { g.src[s] = l.seg[s].src; g.k[s] = l.seg[s].k; }
        g.w_off = woff;
        g.bias_off = foff;
        g.epi = l.epi;
        woff += (g.k[0] + g.k[1]) * g.n * 2;
        foff += layer ? g.n : P.bstride;
    }
    P.plane_bytes = woff;
    P.sigma_w_off = foff;
    P.f32_floats = layer ? foff + pad8(nd.L) + 4 + nd.rgb_dim * pad8(nd.rgb_in) + mn_tc_lg_rgb_bound(nd.rgb_dim) : foff + nd.L + 4;
    P.f32_off = woff * 2;
    P.sub_bytes = (int)mn_align((size_t)woff * 2 + (size_t)P.f32_floats * 4, 256);
    P.x_tile_bytes = (P.kpe + P.kaux) * kTileM * 2;
}

// ---- data-gradient chain of the backward (training, needs dir_a_encoding): dX of every Linear from dir_a_encoding down to trunk
// layer 1, restricted to its L hidden input columns, each a GEMM on the Linear's transposed weight image [N/256][K/8][256][8]
// fp16 (at L = 256 the [K/8][N][8] image of the fused kernel), N = the hidden input columns, K = the Linear's output columns.
// On the layer engine K is the width of the output's gradient image (TcLinear::cols) and N is padded to 256-column blocks,
// both with zero weights.  The images follow each other in that order, then the fp32 block [sigma_w (hc)][rgb_w [rgb_dim][L/2]]
// (sigma_w zero-padded to the H image's columns, which the layer engine's dsigma epilogue reads).  The fused engine runs the plan
// in tc_mlp_wg_kernel<PP_DGRAD>; the layer engine reads the images' offsets from it (one tc_layer_gemm_kernel<false, true>
// launch each) and ignores rgb_w.
void build_dgrad_plan(const NetDims& nd, const TcLinears& T, bool layer, TcPlan* p) {
    TcPlan& P = *p;
    P = TcPlan{};
    P.L = nd.L;
    P.bstride = 256;
    int woff = 0, ng = 0;
    for (int j = T.n - 2; j >= 1; --j) {     // T.l[T.n - 1] is the rgb Linear: its input gradient comes from the head stage
        const int epi = T.l[j - 1].epi;      // of the Linear whose output gradient this GEMM produces (tape image j - 1)
        TcGemm& g = P.g[ng++];
        g.n = layer ? (nd.L + 255) / 256 * 256 : nd.L;
        g.nseg = 1;
        g.src[0] = SRC_H;
        g.k[0] = T.l[j].cols;
        g.w_off = woff;
        g.img = j - 1;
        g.epi = epi == EPI_LINEAR ? EPI_D_LINEAR : epi == EPI_RELU_SIGMA ? EPI_D_MASK_SIGMA : EPI_D_MASK;
        woff += g.k[0] * g.n * 2;
    }
    P.n_gemm = P.n_trunk = ng;
    P.plane_bytes = woff;
    P.sigma_w_off = 0;
    P.f32_floats = T.hc + nd.rgb_dim * (nd.L / 2);
    P.f32_off = woff;
    P.sub_bytes = (int)mn_align((size_t)woff + (size_t)P.f32_floats * 4, 256);
}

LgNet lg_net(const TcNet& net, const NetDims& nd) {
    const TcPlan& P = net.P;
    LgNet b{};
    b.g_gemm = nd.has_dir_a ? P.n_gemm - 1 : -1;
    b.buf_cols[LB_ACT0] = b.buf_cols[LB_ACT1] = net.lin.hc;
    if (nd.has_dir_a) b.buf_cols[LB_G] = net.lin.gc;
    b.h_last = (nd.layers - 1) & 1;
    b.rgb_src = nd.has_dir_a ? LB_G : b.h_last;
    b.sigma_k = pad8(nd.L);
    b.rgb_k = pad8(nd.rgb_in);
    b.rgb_w_off = P.sigma_w_off + b.sigma_k + 4;
    b.rgb_b_off = b.rgb_w_off + nd.rgb_dim * b.rgb_k;
    return b;
}

// ------------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded wait: a protocol bug becomes a trap (launch failure) instead of a hung GPU.  No printf here: a function call
// between an asynchronous warpgroup MMA and its wait makes the compiler serialise every wgmma.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    if (mbar_try(bar, parity)) return;
    const long long t0 = clock64();
    while (!mbar_try(bar, parity)) {
        if (clock64() - t0 > 4000000000ll) __trap();
    }
}
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
    const __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h);
}


// rgb head epilogue shared by the tensor-core kernels (nerf.py:152-160): bias, optional per-image affine appearance
// transform (3x4 matrix = affine(embedding_a[idx]), nerf.py:156-158), sigmoid when rgb_dim == 3, blend weight.
// v = the row's raw fp32 accumulators of the rgb Linear, kR >= rgb_dim of them; bias = NULL when they include the bias
// (the fused kernel's rgb GEMM starts its accumulators at it).
template <int kR = MN_TC_RGB_MAX>
__device__ __forceinline__ void tc_emit_rgb(const MlpArgs& m, int sub, int64_t row, int64_t slot, const uint32_t* v,
                                            const float* bias, float sigma, float* tape_rgb = nullptr) {
    const NetDims& nd = m.nd;
    const int64_t o = (m.scatter ? row : slot) * m.out_cols;
    const float w = m.slot_w ? m.slot_w[slot] : 1.0f;
    if (nd.affine && nd.app > 0) {
        const float* Pk = m.packed + (size_t)sub * m.lay.total;
        const float* emb = Pk + m.lay.emb;
        const float* aw = Pk + m.lay.aff_w;   // [app][12]
        int id = (int)m.src.index(row);
        id = min(max(id, 0), nd.app_count - 1);
        float T[12];
#pragma unroll
        for (int q = 0; q < 12; ++q) T[q] = Pk[m.lay.aff_b + q];
        for (int j = 0; j < nd.app; ++j) {
            const float e = emb[(size_t)id * nd.app + j];
#pragma unroll
            for (int q = 0; q < 12; ++q) T[q] = fmaf(e, aw[j * 12 + q], T[q]);
        }
        float r0 = __uint_as_float(v[0]), r1 = __uint_as_float(v[1]), r2 = __uint_as_float(v[2]);
        if (bias) { r0 = r0 + bias[0]; r1 = r1 + bias[1]; r2 = r2 + bias[2]; }
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float x = mn_sigmoid(fmaf(T[c * 4 + 2], r2, fmaf(T[c * 4 + 1], r1, T[c * 4 + 0] * r0)) + T[c * 4 + 3]);
            m.out[o + c] = m.slot_w ? x * w : x;
        }
    } else {
#pragma unroll
        for (int c = 0; c < kR; ++c) {
            if (c < nd.rgb_dim) {
                float x = __uint_as_float(v[c]);
                if (bias) x = x + bias[c];
                if (nd.rgb_dim == 3) x = mn_sigmoid(x);
                if (tape_rgb && c < 3) tape_rgb[c * kTileM] = x;      // training forward: colour before the blend weight
                m.out[o + c] = m.slot_w ? x * w : x;
            }
        }
    }
    m.out[o + nd.rgb_dim] = m.slot_w ? sigma * w : sigma;
}

// ------------------------------------------------------------------------------------------------
// feature tiles
// ------------------------------------------------------------------------------------------------
// Feature tiles tile0 .. tile0 + gridDim.x - 1 (global index: routing, rows), stored from tile 0 of ximg: the fused engine
// encodes every tile in one launch (tile0 = 0), the layer-GEMM engine one tile group per launch.
__global__ void __launch_bounds__(kTileM) tc_encode_kernel(const MlpArgs a, int kpe, int kaux, int split, __half* __restrict__ ximg,
                                                           int64_t plane_stride_halves, int64_t tile0) {
    const int64_t tile = tile0 + blockIdx.x, out_tile = blockIdx.x;
    extern __shared__ __align__(16) unsigned char sm_raw[];
    __half* img = reinterpret_cast<__half*>(sm_raw);                  // hi image, then lo image
    const int ktot = kpe + kaux;
    const NetDims& nd = a.nd;
    const int t = threadIdx.x;
    const int64_t slot0 = tile * kTileM;
    const int64_t n_slots = a.n_slots();
    if (slot0 >= n_slots) return;
    const int64_t row = a.row_of_slot(slot0 + t, n_slots);
    __half* lo_img = img + (size_t)ktot * kTileM;
    auto put = [&](int col, float v) {
        const int o = (col >> 3) * (kTileM * 8) + t * 8 + (col & 7);
        const __half h = __float2half_rn(v);
        img[o] = h;
        if (split) lo_img[o] = __float2half_rn(v - __half2float(h));
    };
    const int sub = a.sub_of_tile(tile);
    if (row < 0) {
        for (int c = 0; c < ktot; ++c) put(c, 0.0f);
    } else {
        float x[4];
        for (int j = 0; j < nd.xyz_dim; ++j) { x[j] = a.src.xyz(row, j); put(j, x[j]); }
        for (int k = 0; k < nd.nf_xyz; ++k)
            for (int j = 0; j < nd.xyz_dim; ++j) {
                float s, c;
                mn_pe_sincos(x[j], k, &s, &c);
                const int base = nd.xyz_dim + k * 2 * nd.xyz_dim;
                put(base + j, s);
                put(base + nd.xyz_dim + j, c);
            }
        for (int c = nd.in_xyz; c < kpe; ++c) put(c, 0.0f);
        if (kaux > 0) {
            int col = kpe;
            if (!a.sigma_only) {
                if (nd.nf_dir > 0) {
                    float d[3];
                    for (int j = 0; j < 3; ++j) { d[j] = a.src.dir(row, j); put(col + j, d[j]); }
                    for (int k = 0; k < nd.nf_dir; ++k)
                        for (int j = 0; j < 3; ++j) {
                            float s, c;
                            mn_pe_sincos(d[j], k, &s, &c);
                            put(col + 3 + k * 6 + j, s);
                            put(col + 3 + k * 6 + 3 + j, c);
                        }
                    col += nd.in_dir;
                }
                if (nd.app_in_dira) {
                    const float* emb = a.packed + (size_t)sub * a.lay.total + a.lay.emb;
                    int id = (int)a.src.index(row);
                    id = min(max(id, 0), nd.app_count - 1);
                    for (int j = 0; j < nd.app; ++j) put(col + j, emb[(size_t)id * nd.app + j]);
                    col += nd.app;
                }
            }
            for (int c = col; c < ktot; ++c) put(c, 0.0f);
        }
    }
    __syncthreads();
    const int nvec = ktot * kTileM * 2 / 16;
    const uint4* s4 = reinterpret_cast<const uint4*>(img);
    uint4* d4 = reinterpret_cast<uint4*>(ximg + out_tile * (int64_t)ktot * kTileM);
    for (int i = t; i < nvec; i += kTileM) d4[i] = s4[i];
    if (split) {
        const uint4* s4l = reinterpret_cast<const uint4*>(lo_img);
        uint4* d4l = reinterpret_cast<uint4*>(ximg + plane_stride_halves + out_tile * (int64_t)ktot * kTileM);
        for (int i = t; i < nvec; i += kTileM) d4l[i] = s4l[i];
    }
}


// sin / cos of 2^k x for consecutive k (nerf.py:19-25): every fourth band is evaluated with the accurate sincosf, the
// three bands after it by the double-angle identities.  A doubling can multiply the absolute error by up to 6 (the sine's
// error feeds the cosine's and back), so the result is not a few ulps away: tests/test_tc_train_ref.py measures up to 1.4e-6
// (about 24 fp32 ulps at 1) from the directly evaluated value - still two orders of magnitude below the fp16 rounding
// (2.4e-4) these features undergo on their way into the tensor-core operand tile.  (s, c) carry band k-1 in.
__device__ __forceinline__ void pe_band(float x, int k, float* s, float* c) {
    if ((k & 3) == 0) {
        mn_pe_sincos(x, k, s, c);
    } else {
        const float s0 = *s, c0 = *c;
        *s = 2.0f * s0 * c0;
        *c = 1.0f - 2.0f * s0 * s0;
    }
}

// Specialised encoder for the common network shape (compile-time channel counts): every thread builds its row's
// channels in registers and writes the tile image straight to global memory with 16-byte stores (thread t of a
// chunk writes bytes [t*16, t*16+16) -> fully coalesced); no shared-memory staging, no 2-byte bank-conflicted stores.
template <int XD, int NFX, int NFD, int APP>
__global__ void __launch_bounds__(kTileM) tc_encode_fast_kernel(const MlpArgs a, __half* __restrict__ ximg) {
    constexpr int IN_XYZ = XD * (1 + 2 * NFX);
    constexpr int KPE = (IN_XYZ + 15) / 16 * 16;
    constexpr int IN_DIR = NFD > 0 ? 3 + 6 * NFD : 0;
    constexpr int KAUX = (IN_DIR + APP + 15) / 16 * 16;
    const int t = threadIdx.x;
    const int64_t tile = blockIdx.x;
    const int64_t slot0 = tile * kTileM;
    const int64_t n_slots = a.n_slots();
    if (slot0 >= n_slots) return;
    const int64_t row = a.row_of_slot(slot0 + t, n_slots);
    uint4* out = reinterpret_cast<uint4*>(ximg + tile * (int64_t)(KPE + KAUX) * kTileM) + t;   // + chunk * kTileM
    {
        float v[KPE];
#pragma unroll
        for (int c = 0; c < KPE; ++c) v[c] = 0.0f;
        if (row >= 0) {
#pragma unroll
            for (int j = 0; j < XD; ++j) {
                const float x = a.src.xyz(row, j);
                v[j] = x;
                float s = 0.0f, c = 1.0f;
#pragma unroll
                for (int k = 0; k < NFX; ++k) {
                    pe_band(x, k, &s, &c);
                    v[XD + k * 2 * XD + j] = s;
                    v[XD + k * 2 * XD + XD + j] = c;
                }
            }
        }
#pragma unroll
        for (int c = 0; c < KPE / 8; ++c)
            out[c * kTileM] = make_uint4(pack_h2(v[8 * c], v[8 * c + 1]), pack_h2(v[8 * c + 2], v[8 * c + 3]),
                                         pack_h2(v[8 * c + 4], v[8 * c + 5]), pack_h2(v[8 * c + 6], v[8 * c + 7]));
    }
    if (KAUX > 0) {
        float v[KAUX > 0 ? KAUX : 1];
#pragma unroll
        for (int c = 0; c < KAUX; ++c) v[c] = 0.0f;
        if (row >= 0 && !a.sigma_only) {
            if (NFD > 0) {
#pragma unroll
                for (int j = 0; j < 3; ++j) {
                    const float d = a.src.dir(row, j);
                    v[j] = d;
                    float s = 0.0f, c = 1.0f;
#pragma unroll
                    for (int k = 0; k < NFD; ++k) {
                        pe_band(d, k, &s, &c);
                        v[3 + k * 6 + j] = s;
                        v[3 + k * 6 + 3 + j] = c;
                    }
                }
            }
            if (APP > 0) {
                const int sub = a.sub_of_tile(tile);
                int id = (int)a.src.index(row);
                id = min(max(id, 0), a.nd.app_count - 1);
                const float4* e4 = reinterpret_cast<const float4*>(a.packed + (size_t)sub * a.lay.total + a.lay.emb + (size_t)id * APP);
#pragma unroll
                for (int j = 0; j < APP / 4; ++j) {
                    const float4 e = __ldg(e4 + j);
                    v[IN_DIR + 4 * j + 0] = e.x;
                    v[IN_DIR + 4 * j + 1] = e.y;
                    v[IN_DIR + 4 * j + 2] = e.z;
                    v[IN_DIR + 4 * j + 3] = e.w;
                }
            }
        }
#pragma unroll
        for (int c = 0; c < KAUX / 8; ++c)
            out[(KPE / 8 + c) * kTileM] = make_uint4(pack_h2(v[8 * c], v[8 * c + 1]), pack_h2(v[8 * c + 2], v[8 * c + 3]),
                                                     pack_h2(v[8 * c + 4], v[8 * c + 5]), pack_h2(v[8 * c + 6], v[8 * c + 7]));
    }
}



// ------------------------------------------------------------------------------------------------
// the MLP kernel
// ------------------------------------------------------------------------------------------------
struct TcArgs {
    MlpArgs m;
    TcPlan plan;
    const unsigned char* wpack;   // per sub-module: [hi plane][lo plane?][fp32 block]
    const __half* ximg;           // feature tiles (hi plane; lo plane at +x_plane_halves)
    int64_t x_plane_halves;
    int split;                    // 1: three MMA passes (hi*hi + hi*lo + lo*hi)
    int64_t n_tiles_cap;
    // ---- training (tc_f16 training path, mn_train_tc.cuh).  Per 128-slot tile, records of fp16 tile images (mn_model.cuh,
    // mn_tc_img_off) and fp32 head blocks.
    unsigned char* tape_act;      // PP_TRAIN_FWD: written;  PP_DGRAD: read (ReLU masks)
    float* tape_f32;              // fp32 head blocks [MN_TC_F32_ROWS][128]     (written / read)
    unsigned char* tape_dz;       // PP_DGRAD: gradient images dZ_0 .. dZ_{layers-1}, dZ_final, dZ_dira (same layout, scaled fp16)
    float* tape_gf32;             // PP_DGRAD: head-gradient blocks [mn_tc_g32_rows(rgb_dim)][128], UNscaled fp32
    const float* grad_out;        // PP_DGRAD: [rows][rgb_dim + 1] upstream gradient
    float* emb_sum;               // PP_DGRAD: [n_sub][app_count][L/2] per-image sums of dZ_dira rows (appearance-embedding gradient)
    const float* scale;           // PP_DGRAD: device scalar S (power of two): gradient images hold S * dZ
    int64_t act_tile_bytes;       // bytes of one tile's record in tape_act / tape_dz
    int layers;
};

constexpr int kSmemMax = 227 * 1024;

#include "mn_mlp_wg.cuh"

// The variant of tc_mlp_wg_kernel that runs mode over plan P, and its shared-memory layout; split (tc_f16x3): inference <= 256 wide.
struct WgVariant {
    void (*kernel)(TcArgs);
    WgLayout layout;
};
WgVariant wg_variant(int mode, bool split, const TcPlan& P) {
    const bool wide = P.L > 256;
    static void (*const kernel[3][2])(TcArgs) = {       // [mode][wide]
        {tc_mlp_wg_kernel<PP_INFER, false, false>, tc_mlp_wg_kernel<PP_INFER, false, true>},
        {tc_mlp_wg_kernel<PP_TRAIN_FWD, false, false>, tc_mlp_wg_kernel<PP_TRAIN_FWD, false, true>},
        {tc_mlp_wg_kernel<PP_DGRAD, false, false>, tc_mlp_wg_kernel<PP_DGRAD, false, true>}};
    return {split ? tc_mlp_wg_kernel<PP_INFER, true, false> : kernel[mode][wide], wg_layout(P, split, wg_reg_act(mode, split, wide))};
}

int wg_launch(mn_ctx* ctx, const TcArgs& A, int mode, int64_t n_tiles128, cudaStream_t st) {
    const auto [kernel, WL] = wg_variant(mode, A.split, A.plan);
    if (WL.total > kSmemMax || WL.stages < 2) return mn_fail(ctx, MN_ERR_UNSUPPORTED, "tensor-core MLP: shared-memory budget exceeded");
    MN_CUDA(ctx, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, WL.total));
    const unsigned grid = (unsigned)(n_tiles128 < ctx->sm_count ? n_tiles128 : ctx->sm_count);
    kernel<<<grid, kWgmmaThreads, WL.total, st>>>(A);
    MN_LAUNCH_CHECK(ctx);
    return MN_OK;
}

#include "mn_train_tc.cuh"
#include "mn_layer_gemm.cuh"

// Workspace of a forward call: per tile of a group, the feature tile and the layer engine's activation buffers, each with its lo
// plane under tc_f16x3.  The fused engine's one group covers every tile and has no activation buffers; the layer engine's
// groups are bounded by kLgGroupTiles, not by the call's rows.
struct TcWorkspace {
    int64_t group_tiles;
    size_t x_bytes, buf_bytes[3], total;     // per plane
    int planes;
};
TcWorkspace tc_workspace(const TcNet& net, int64_t n_tiles128, int precision) {
    TcWorkspace w{};
    w.group_tiles = net.engine == TC_LAYER && n_tiles128 > kLgGroupTiles ? kLgGroupTiles : n_tiles128;
    w.planes = precision == MN_PREC_TC_F16X3 ? 2 : 1;
    w.x_bytes = mn_align((size_t)w.group_tiles * net.P.x_tile_bytes, 1024);
    w.total = w.x_bytes * w.planes;
    for (int b = 0; b < 3; ++b) {
        w.buf_bytes[b] = mn_align((size_t)w.group_tiles * net.lg.buf_cols[b] * kTileM * 2, 1024);
        w.total += w.buf_bytes[b] * w.planes;
    }
    w.total += 1024;
    return w;
}

// A tile image that a layer GEMM reads or writes: tile 0 of the group, the tile stride, the lo plane's offset (0: none).
struct LgImg {
    unsigned char* p;
    int64_t tile_bytes, lo;
};

// One tc_layer_gemm_kernel launch of GEMM g of plan P (weights at wpack) over the tiles t0 .. t0 + nt - 1 of a group, storing its
// first n_out columns to out.  A segment reads x (SRC_XPE / SRC_XAUX: the feature tile) or h (SRC_H).  G carries what the forward
// and the data-gradient GEMMs do not share: bias and ReLU, or mask, dsig and scale.
int lg_gemm(mn_ctx* ctx, LgArgs G, const MlpArgs& a, const TcPlan& P, const TcGemm& g, const void* wpack, int n_out, int64_t t0,
            int64_t nt, LgImg x, LgImg h, LgImg out, bool split, bool dgrad, cudaStream_t st) {
    G.m = a;
    G.tile0 = t0;
    G.n_tiles = nt;
    G.wpack = (const unsigned char*)wpack;
    G.sub_bytes = P.sub_bytes;
    G.w_off = g.w_off;
    G.k_tot = g.k[0] + (g.nseg > 1 ? g.k[1] : 0);
    G.n_blk = g.n / kLgBlock;
    G.n_out = n_out;
    G.f32_off = P.f32_off;
    G.nseg = g.nseg;
    for (int s = 0; s < g.nseg; ++s) {
        const LgImg& in = g.src[s] == SRC_H ? h : x;
        G.a[s] = in.p + (g.src[s] == SRC_XAUX ? P.kpe * kTileM * 2 : 0);
        G.ak[s] = g.k[s];
        G.a_tile_bytes[s] = in.tile_bytes;
        G.a_lo[s] = in.lo;
    }
    G.out = out.p;
    G.out_tile_bytes = out.tile_bytes;
    G.out_lo = out.lo;
    const int64_t items = nt * G.n_blk;
    const unsigned grid = (unsigned)(items < ctx->sm_count ? items : ctx->sm_count);
    auto launch = [&](auto kernel, int smem) -> int {
        MN_CUDA(ctx, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        kernel<<<grid, kWgmmaThreads, smem, st>>>(G);
        MN_LAUNCH_CHECK(ctx);
        return MN_OK;
    };
    if (dgrad) return launch(tc_layer_gemm_kernel<false, true>, LgShape<false>::smem);
    if (split) return launch(tc_layer_gemm_kernel<true>, LgShape<true>::smem);
    return launch(tc_layer_gemm_kernel<false>, LgShape<false>::smem);
}

}  // namespace

// =================================================================================================
size_t mn_mlp_tc_workspace(const mn_model* m, int64_t n_tiles128, int precision) {
    return m->tc.engine == TC_NONE ? 0 : tc_workspace(m->tc, n_tiles128, precision).total;
}

// ---- which engine serves a network, and whether tensor-core training covers it.  The fused engine takes rgb_dim <= 32 (its
// N = 32 rgb GEMM) at 64..256 (a multiple of 64) and 512 wide, up to 12 trunk layers; the layer engine every other width of
// 64..kLgMaxL and depth (up to MN_MAX_LAYERS), and the SH heads of degree 3 and 4 (rgb_dim <= MN_TC_LG_RGB_MAX).  Training
// runs on the fused engine at 256 and 512 wide (every depth it takes, 2..12 trunk layers) and on the layer engine from 256
// wide; it needs dir_a_encoding (its data-gradient chain ends there) and no affine appearance.  A network is trained on the
// engine that runs its inference, so the recording forward writes the tape that engine's backward reads.
// Defined after mn_mlp_tc_workspace: nvcc names the anonymous namespace, so every kernel, after the first function outside it.
constexpr int kLgMaxL = 4096;
TcNet tc_net(const mn_model& m) {
    const NetDims& nd = m.nd;
    TcNet t{};
    const bool fused_width = nd.L % 64 == 0 && (nd.L <= 256 || nd.L == 512) && nd.L >= 64;
    if (nd.affine && nd.rgb_dim != 3) t.engine = TC_NONE;
    else if (fused_width && nd.rgb_dim <= MN_TC_RGB_MAX && nd.layers <= 12)
        t.engine = TC_FUSED;
    else if (nd.L >= 64 && nd.L <= kLgMaxL && nd.rgb_dim <= MN_TC_LG_RGB_MAX && nd.layers + 2 <= kMaxGemm)
        t.engine = TC_LAYER;
    const bool layer = t.engine == TC_LAYER;
    t.lin = tc_linears(m, layer);
    if (t.engine != TC_NONE) build_plan(nd, t.lin, layer, &t.P);
    if (layer) t.lg = lg_net(t, nd);
    t.train = nd.has_dir_a && !nd.affine && nd.rgb_dim >= 3 && nd.layers >= 2 &&
              ((layer && nd.L >= 256) || (t.engine == TC_FUSED && (nd.L == 256 || nd.L == 512) && nd.layers <= 12));
    if (t.train) build_dgrad_plan(nd, t.lin, layer, &t.D);
    t.act_tile_bytes = (int64_t)(mn_tc_img_off(nd.layers + 1, t.lin.hc) + mn_tc_img_off(1, t.lin.gc));     // ends with G (L/2 columns)
    return t;
}

// mode: PP_INFER (the tc_f16 inference launch), PP_TRAIN_FWD (the recording forward: the forward plan in the training variant's
// layout) or PP_DGRAD (the data-gradient chain of the backward on the transposed images); the training modes only for shapes
// whose training runs on the fused engine.
int mn_mlp_tp_program(const mn_model& m, int mode, unsigned int* table_out, int cap_entries, int* info8) {
    const TcNet& net = m.tc;
    if (net.engine != TC_FUSED || (mode != PP_INFER && !net.train)) return MN_ERR_UNSUPPORTED;
    const TcPlan& P = mode == PP_DGRAD ? net.D : net.P;
    const WgLayout L = wg_variant(mode, false, P).layout;     // the tc_f16 launch's layout
    int n = 0, n_trunk = 0;
    for (int gi = 0; gi < P.n_gemm; ++gi) {
        const int nch = (P.g[gi].n + 255) >> 8;
        for (int ch = 0; ch < nch; ++ch)
            wg_walk_chunk(P, gi, ch, 1, L.slab, [&](const WgStage& st) {
                if (n < cap_entries) {
                    unsigned int* e = table_out + 8 * (size_t)n;
                    e[0] = (unsigned)st.w_off; e[1] = (unsigned)st.w_bytes; e[2] = (unsigned)st.nw; e[3] = (unsigned)st.kc;
                    e[4] = (unsigned)st.a_col; e[5] = (unsigned)st.x_off; e[6] = (unsigned)st.x_bytes;
                    e[7] = (unsigned)st.flags | ((unsigned)gi << 8) | ((unsigned)ch << 16);
                }
                ++n;
            });
        if (gi + 1 == P.n_trunk) n_trunk = n;
    }
    const int info[8] = {n, n_trunk, P.plane_bytes, L.stages, L.total, P.x_tile_bytes, L.stage_bytes, L.slab};
    for (int i = 0; i < 8; ++i) info8[i] = info[i];
    return n <= cap_entries ? MN_OK : MN_ERR_WORKSPACE;
}

// ---- transposed weight images of the data-gradient chain (build_dgrad_plan), one fp16 plane + the fp32 block per sub-module.
// Element (n = input column, k = output channel) = W[k][n]: the [out][L] BwdLayout sub-matrix is the K-major source.
static void tc_pack_dgrad(mn_ctx* ctx, mn_model* m, int sub) {
    const NetDims& nd = m->nd;
    const TcPlan& D = m->tc.D;
    unsigned char* db = (unsigned char*)m->tc_dgrad + (size_t)sub * D.sub_bytes;
    const float* Q = m->packed_bwd + (size_t)sub * m->blay.total;
    const float* Pk = m->packed + (size_t)sub * m->lay.total;
    for (int gi = 0; gi < D.n_gemm; ++gi) {
        const TcGemm& g = D.g[gi];
        const TcLinear& l = m->tc.lin.l[g.img + 1];
        const int k = g.k[0];          // l.cols: the output channels past l.n are zero rows of the image
        mn_pack_push(ctx, PackOp{Q + l.bwd, db + g.w_off, nullptr, (long long)g.n * k, PK_TC_HALF, {nd.L, l.n, g.n, k, 0, 0, 256}});
    }
    float* f32 = reinterpret_cast<float*>(db + D.f32_off);
    mn_pack_push(ctx, PackOp{Pk + m->lay.sigma_w, f32, nullptr, (long long)nd.L, PK_TC_F32, {nd.L, 0, 0, 0, 0, 0, 0}});
    mn_pack_push(ctx, PackOp{Pk + m->lay.rgb_w, f32 + m->tc.lin.hc, nullptr, (long long)nd.rgb_dim * (nd.L / 2), PK_RGBW,
                             {nd.L / 2, nd.rgb_dim, 0, 0, 0, 0, 0}});
}

// The transposed images cost as much as the forward images again, so they are allocated and packed by the first recording call
// (inference-only users never hold them); from then on every mn_model_set_weights repacks them with the forward images.
static int tc_dgrad_ready(mn_ctx* ctx, mn_model* m, cudaStream_t st) {
    if (m->tc_dgrad) return MN_OK;
    const size_t bytes = (size_t)m->tc.D.sub_bytes * m->d.n_sub;
    MN_CUDA(ctx, cudaMalloc(&m->tc_dgrad, bytes));
    MN_CUDA(ctx, cudaMemsetAsync(m->tc_dgrad, 0, bytes, st));
    for (int s = 0; s < m->d.n_sub; ++s) tc_pack_dgrad(ctx, m, s);
    return mn_pack_flush(ctx, st);
}

// Forward weight images.  Per sub-module: [hi plane][lo plane][fp32 block], every weight image [N/nw][K/8][nw][8] fp16 with its
// fp16 residual in the lo plane: nw = N <= 256 for the fused engine (two N = 256 halves for the 512-wide network), 256 for the
// layer engine (its N is padded to 256-column blocks).  The fp32 block holds the biases, sigma_w and sigma_b, and for the layer
// engine the rgb head.  Queued: all images of the sub-module are written by ONE launch (mn_pack_flush in mn_model_set_weights).
int mn_mlp_tc_pack(mn_ctx* ctx, mn_model* m, int sub, cudaStream_t st) {
    const TcNet& net = m->tc;
    if (net.engine == TC_NONE) return MN_OK;  // configuration only served by the fp32 kernel
    const NetDims& nd = m->nd;
    const TcPlan& P = net.P;
    const size_t sub_bytes = (size_t)P.sub_bytes;
    if (!m->tc_packed) {
        MN_CUDA(ctx, cudaMalloc(&m->tc_packed, sub_bytes * m->d.n_sub));
        MN_CUDA(ctx, cudaMemsetAsync(m->tc_packed, 0, sub_bytes * m->d.n_sub, st));
    }
    unsigned char* base = (unsigned char*)m->tc_packed + (size_t)sub * sub_bytes;
    const float* Pk = m->packed + (size_t)sub * m->lay.total;
    float* f32 = reinterpret_cast<float*>(base + P.f32_off);
    for (int gi = 0; gi < P.n_gemm; ++gi) {
        const TcLinear& l = net.lin.l[gi];
        const TcGemm& g = P.g[gi];
        const int K = g.k[0] + g.k[1];
        // the leading segment holds its real columns, then zeros up to its padded width; the second segment's columns follow
        // contiguously, and columns past in_features (the padding of a second H segment) are zero
        mn_pack_push(ctx, PackOp{Pk + l.w, base + g.w_off, base + P.plane_bytes + g.w_off, (long long)g.n * K, PK_TC_HALF,
                                 {l.n, l.kin, g.n, K, l.seg[0].k_real, l.seg[0].k, g.n < 256 ? g.n : 256}});
        // the bias fills the floats the plan reserved for it, up to the next bias (sigma_w after the last one)
        const int b_end = gi + 1 < P.n_gemm ? P.g[gi + 1].bias_off : P.sigma_w_off;
        mn_pack_push(ctx, PackOp{Pk + l.b, f32 + g.bias_off, nullptr, (long long)(b_end - g.bias_off), PK_TC_F32, {l.n, 0, 0, 0, 0, 0, 0}});
    }
    const bool layer = net.engine == TC_LAYER;
    const LgNet& B = net.lg;
    const int sigma_k = layer ? B.sigma_k : nd.L;
    mn_pack_push(ctx, PackOp{Pk + m->lay.sigma_w, f32 + P.sigma_w_off, nullptr, (long long)nd.L, PK_TC_F32, {nd.L, 0, 0, 0, 0, 0, 0}});
    mn_pack_push(ctx, PackOp{Pk + m->lay.sigma_b, f32 + P.sigma_w_off + sigma_k, nullptr, 4, PK_TC_F32, {1, 0, 0, 0, 0, 0, 0}});
    if (layer) {      // tc_layer_head_kernel computes the rgb head on the CUDA cores
        mn_pack_push(ctx, PackOp{Pk + m->lay.rgb_w, f32 + B.rgb_w_off, nullptr, (long long)nd.rgb_dim * nd.rgb_in, PK_RGBW,
                                 {nd.rgb_in, nd.rgb_dim, B.rgb_k, 0, 0, 0, 0}});
        mn_pack_push(ctx, PackOp{Pk + m->lay.rgb_b, f32 + B.rgb_b_off, nullptr, mn_tc_lg_rgb_bound(nd.rgb_dim), PK_TC_F32,
                                 {nd.rgb_dim, 0, 0, 0, 0, 0, 0}});
    }
    if (net.train && m->tc_dgrad) tc_pack_dgrad(ctx, m, sub);
    return MN_OK;
}

// Feature tiles of the first n_tiles128 tiles: the specialised encoder for the common network shape, the generic one otherwise.
static int tc_encode(mn_ctx* ctx, const mn_model* m, const MlpArgs& a, const TcPlan& P, int64_t n_tiles128, int split,
                     __half* ximg, int64_t plane_halves, cudaStream_t st) {
    const size_t enc_sm = (size_t)P.x_tile_bytes * (split ? 2 : 1);
    MN_CUDA(ctx, cudaFuncSetAttribute(tc_encode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)enc_sm));
    const NetDims& nd = a.nd;
    const bool fast_shape = !split && nd.xyz_dim == 3 && nd.nf_xyz == 12 && nd.nf_dir == 4 && nd.app == 48 && nd.app_in_dira &&
                            (m->lay.emb % 4) == 0;
    if (fast_shape)
        tc_encode_fast_kernel<3, 12, 4, 48><<<(unsigned)n_tiles128, kTileM, 0, st>>>(a, ximg);
    else
        tc_encode_kernel<<<(unsigned)n_tiles128, kTileM, enc_sm, st>>>(a, P.kpe, P.kaux, split, ximg, plane_halves, 0);
    MN_LAUNCH_CHECK(ctx);
    return MN_OK;
}

// TcArgs fields common to the inference and the recording forward of the fused engine: the plan and the model's packed weights.
static TcArgs tc_forward_args(const mn_model* m, const TcPlan& F, const MlpArgs& a, int64_t n_tiles128) {
    TcArgs A{};
    A.plan = F;
    A.m = a;
    A.wpack = (const unsigned char*)m->tc_packed;
    A.n_tiles_cap = n_tiles128;
    return A;
}

// Layer-GEMM path: the slot tiles in groups of kLgGroupTiles; per group one encoder launch, one GEMM launch per Linear and one
// head launch.  The group count follows from the slot capacity, so a call is a static launch list (graph capture works).
// tape != NULL (recording call, tc_f16): the encoder tiles, every GEMM's output (image gi of the tile's activation record) and
// the fp32 head blocks go to the tape instead of the workspace, which is not used.
static int layer_launch(mn_ctx* ctx, mn_model* m, const MlpArgs& a, const TcNet& net, int64_t n_tiles128, int precision,
                        void* ws, size_t ws_bytes, cudaStream_t st, const TrainTcTape* tape = nullptr) {
    if (!m->tc_packed) return mn_fail(ctx, MN_ERR_UNSUPPORTED, "tensor-core MLP: weights not packed");
    if (n_tiles128 <= 0) return MN_OK;
    const TcPlan& P = net.P;
    const LgNet& B = net.lg;
    const int hc = net.lin.hc;
    const TcWorkspace W = tc_workspace(net, n_tiles128, precision);
    if (!tape && (ws_bytes < W.total || !ws)) return mn_fail(ctx, MN_ERR_WORKSPACE, "mn_mlp_tc_launch: workspace too small");
    const bool split = precision == MN_PREC_TC_F16X3;
    unsigned char* wp = (unsigned char*)(((uintptr_t)ws + 1023) / 1024 * 1024);
    __half* ximg = reinterpret_cast<__half*>(wp);
    const int64_t x_lo = (int64_t)W.x_bytes;                 // lo plane of each region right after its hi plane
    wp += W.x_bytes * W.planes;
    LgImg buf[3];
    for (int b = 0; b < 3; ++b) {
        buf[b] = LgImg{wp, (int64_t)B.buf_cols[b] * kTileM * 2, (int64_t)W.buf_bytes[b]};
        wp += W.buf_bytes[b] * W.planes;
    }
    const int64_t act_tile = tape ? net.act_tile_bytes : 0;

    const size_t enc_sm = (size_t)P.x_tile_bytes * (split ? 2 : 1);
    MN_CUDA(ctx, cudaFuncSetAttribute(tc_encode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)enc_sm));
    const int n_gemm = a.sigma_only ? P.n_trunk : P.n_gemm;
    const int64_t plane_halves = x_lo / 2;

    mn_prof_begin(ctx, st);
    for (int64_t t0 = 0; t0 < n_tiles128; t0 += W.group_tiles) {
        const int64_t nt = n_tiles128 - t0 < W.group_tiles ? n_tiles128 - t0 : W.group_tiles;
        unsigned char* rec = tape ? tape->act + t0 * act_tile : nullptr;      // activation record of the group's first tile
        if (tape) ximg = reinterpret_cast<__half*>(tape->xreg + t0 * (int64_t)P.x_tile_bytes);
        tc_encode_kernel<<<(unsigned)nt, kTileM, enc_sm, st>>>(a, P.kpe, P.kaux, split ? 1 : 0, ximg, plane_halves, t0);
        MN_LAUNCH_CHECK(ctx);
        const LgImg x{reinterpret_cast<unsigned char*>(ximg), P.x_tile_bytes, x_lo};
        for (int gi = 0; gi < n_gemm; ++gi) {
            const TcGemm& g = P.g[gi];
            LgArgs G{};
            G.w_lo = P.plane_bytes;
            G.bias_off = g.bias_off;
            G.relu = g.epi != EPI_LINEAR;
            LgImg h = buf[B.in(gi)], out = buf[B.out(gi)];
            if (tape) {       // GEMM gi reads image gi - 1 (SRC_H; trunk layer 0 has none) and writes image gi of the activation record
                h = gi > 0 ? LgImg{rec + mn_tc_img_off(gi - 1, hc), act_tile, 0} : LgImg{};
                out = LgImg{rec + mn_tc_img_off(gi, hc), act_tile, 0};
            }
            // every column of the output image, its zero padding included
            const int rc = lg_gemm(ctx, G, a, P, g, m->tc_packed, net.lin.l[gi].cols, t0, nt, x, h, out, split, false, st);
            if (rc) return rc;
        }
        LhArgs H{};
        H.m = a;
        H.tile0 = t0;
        H.wpack = (const unsigned char*)m->tc_packed;
        H.sub_bytes = P.sub_bytes;
        H.f32_off = P.f32_off;
        H.sigma_w_off = P.sigma_w_off;
        H.rgb_w_off = B.rgb_w_off;
        H.rgb_b_off = B.rgb_b_off;
        H.h = buf[B.h_last].p;
        H.h_tile_bytes = buf[B.h_last].tile_bytes;
        H.h_lo = split ? buf[B.h_last].lo : 0;
        H.g = buf[B.rgb_src].p;
        H.g_tile_bytes = buf[B.rgb_src].tile_bytes;
        H.g_lo = split ? buf[B.rgb_src].lo : 0;
        H.L = B.sigma_k;
        H.rgb_in = B.rgb_k;
        if (tape) {      // without dir_a_encoding the rgb head reads the last trunk image, as it reads B.rgb_src above
            H.h = rec + mn_tc_img_off(a.nd.layers - 1, hc);
            H.g = rec + mn_tc_img_off(a.nd.has_dir_a ? a.nd.layers + 1 : a.nd.layers - 1, hc);
            H.h_tile_bytes = H.g_tile_bytes = act_tile;
            H.tape_f32 = tape->f32;
        }
        if (m->nd.rgb_dim <= MN_TC_RGB_MAX) tc_layer_head_kernel<MN_TC_RGB_MAX><<<(unsigned)nt, kTileM, 0, st>>>(H);
        else tc_layer_head_kernel<MN_TC_LG_RGB_MAX><<<(unsigned)nt, kTileM, 0, st>>>(H);
        MN_LAUNCH_CHECK(ctx);
    }
    mn_prof_end(ctx, st);
    return MN_OK;
}

int mn_mlp_tc_launch(mn_ctx* ctx, mn_model* m, const MlpArgs& a, int64_t n_tiles128, int precision, void* ws, size_t ws_bytes,
                     cudaStream_t st) {
    const TcNet& net = m->tc;
    if (net.engine == TC_LAYER) return layer_launch(ctx, m, a, net, n_tiles128, precision, ws, ws_bytes, st);
    if (net.engine != TC_FUSED || !m->tc_packed)
        return mn_fail(ctx, MN_ERR_UNSUPPORTED,
                       "tensor-core MLP path covers layer_dim 64..4096 with up to 16 layers and rgb_dim <= 80 (sh_deg <= 4), without "
                       "affine appearance for rgb_dim > 3; use precision 'fp32' for this model");
    if (a.nd.L > 256 && precision == MN_PREC_TC_F16X3)
        return mn_fail(ctx, MN_ERR_UNSUPPORTED,
                       "precision 'tc_f16x3' covers layer_dim <= 256; use 'tc_f16' or 'fp32' for the 512-wide network");
    if (n_tiles128 <= 0) return MN_OK;
    TcArgs A = tc_forward_args(m, net.P, a, n_tiles128);
    const int split = precision == MN_PREC_TC_F16X3 ? 1 : 0;
    A.split = split;
    const TcWorkspace W = tc_workspace(net, n_tiles128, precision);
    if (ws_bytes < W.total || !ws) return mn_fail(ctx, MN_ERR_WORKSPACE, "mn_mlp_tc_launch: workspace too small");
    uintptr_t wp = ((uintptr_t)ws + 1023) / 1024 * 1024;
    __half* ximg = reinterpret_cast<__half*>(wp);
    A.ximg = ximg;
    A.x_plane_halves = (int64_t)W.x_bytes / 2;
    int rc = tc_encode(ctx, m, a, A.plan, n_tiles128, split, ximg, A.x_plane_halves, st);
    if (rc) return rc;

    mn_prof_begin(ctx, st);
    rc = wg_launch(ctx, A, PP_INFER, n_tiles128, st);
    mn_prof_end(ctx, st);
    return rc;
}

// =================================================================================================
// tensor-core training path: host side (kernels in mn_train_tc.cuh)
// =================================================================================================
// Recording forward of either engine: encoder tiles and every layer's activations land in the caller's tape.  train: a training
// call, whose caller has checked m->tc.train && m->tc_packed; the first one allocates and packs the transposed images of the
// backward pass.  !train: the test hook mn_debug_tc_forward_record, for every network the tensor cores serve, trained there or
// not; it needs no transposed images, so none are allocated.
int mn_mlp_tc_launch_record(mn_ctx* ctx, mn_model* m, const MlpArgs& a, int64_t n_tiles128, const TrainTcTape& tape, bool train,
                            cudaStream_t st) {
    const TcNet& net = m->tc;
    if (!train && (net.engine == TC_NONE || !m->tc_packed))
        return mn_fail(ctx, MN_ERR_UNSUPPORTED, "mn_debug_tc_forward_record: the network has no tensor-core forward");
    if (n_tiles128 <= 0) return MN_OK;
    int rc;
    if (train && (rc = tc_dgrad_ready(ctx, m, st))) return rc;
    if (net.engine == TC_LAYER) return layer_launch(ctx, m, a, net, n_tiles128, MN_PREC_TC_F16, nullptr, 0, st, &tape);
    TcArgs A = tc_forward_args(m, net.P, a, n_tiles128);
    A.ximg = reinterpret_cast<const __half*>(tape.xreg);
    A.x_plane_halves = 0;
    A.tape_act = tape.act;
    A.tape_f32 = tape.f32;
    A.act_tile_bytes = net.act_tile_bytes;
    A.layers = a.nd.layers;
    if ((rc = tc_encode(ctx, m, a, A.plan, n_tiles128, 0, reinterpret_cast<__half*>(tape.xreg), 0, st))) return rc;
    mn_prof_begin(ctx, st);
    rc = wg_launch(ctx, A, PP_TRAIN_FWD, n_tiles128, st);
    mn_prof_end(ctx, st);
    return rc;
}

// backward workspace: [gradient images][head gradients fp32 [head_tiles][mn_tc_g32_rows(rgb_dim)][128]][embedding sums][scale,
// max |grad_out|].  Fused engine: the gradient records of every tile.  Layer engine: the gradient images of one tile group only
// (dZ_G and two ping-pong H-image-wide buffers), so its workspace is bounded by kLgGroupTiles, not by the row count.  The
// embedding sums are [n_sub][app_count][emb_k] (emb_k: L/2, rounded up to 8 on the layer engine, whose head stage writes whole
// groups of 8 columns).
struct TcBwdWorkspace {
    int64_t head_tiles;
    int emb_k;
    size_t dz_bytes, head_bytes, emb_floats, total;
};
static TcBwdWorkspace tc_bwd_workspace(const mn_model* m, const TcNet& net, int64_t n_tiles128) {
    const NetDims& nd = m->nd;
    TcBwdWorkspace w{};
    w.emb_k = nd.L / 2;
    if (net.engine == TC_LAYER) {
        w.head_tiles = n_tiles128 < kLgGroupTiles ? n_tiles128 : kLgGroupTiles;
        w.dz_bytes = mn_align((size_t)w.head_tiles * net.lin.gc * kTileM * 2) + 2 * mn_align((size_t)w.head_tiles * net.lin.hc * kTileM * 2);
        w.emb_k = pad8(nd.L / 2);
    } else {
        w.head_tiles = n_tiles128;
        w.dz_bytes = mn_align((size_t)n_tiles128 * net.act_tile_bytes);
    }
    w.head_bytes = mn_align((size_t)w.head_tiles * mn_tc_g32_rows(nd.rgb_dim) * kTileM * sizeof(float));
    w.emb_floats = nd.app_in_dira ? (size_t)m->d.n_sub * nd.app_count * w.emb_k : 0;
    w.total = w.dz_bytes + w.head_bytes + mn_align(w.emb_floats * sizeof(float) + 256) + 1024;
    return w;
}
size_t mn_train_tc_backward_workspace(const mn_model* m, int64_t n_tiles128) {
    return tc_bwd_workspace(m, m->tc, n_tiles128).total;
}

// Test hook (mn_debug_tc_train_layout): entries MN_TCL_ENGINE .. of the layout the two training passes share, from the same
// plan (mn_model::tc) and tc_bwd_workspace the passes read.  Backward-workspace offsets are relative to the 256-byte aligned
// base that mn_train_tc_backward carves.
int mn_train_tc_layout(const mn_model* m, int64_t n_tiles128, int64_t* out, int cap) {
    const TcNet& net = m->tc;
    const NetDims& nd = m->nd;
    const int n_img = nd.has_dir_a ? nd.layers + 2 : nd.layers;      // without dir_a_encoding the record holds the trunk only
    if (cap < MN_TCL_IMG + 2 * n_img) return MN_ERR_WORKSPACE;
    out[MN_TCL_ENGINE] = net.engine;
    out[MN_TCL_TRAIN] = net.train ? 1 : 0;
    out[MN_TCL_X_TILE] = net.P.x_tile_bytes;
    out[MN_TCL_ACT_TILE] = net.act_tile_bytes;
    out[MN_TCL_KPE] = net.lin.kpe;
    out[MN_TCL_KAUX] = net.lin.kaux;
    out[MN_TCL_HC] = net.lin.hc;
    out[MN_TCL_GC] = net.lin.gc;
    out[MN_TCL_F32_SIGMA] = MN_TC_F32_SIGMA;
    out[MN_TCL_F32_RGB] = MN_TC_F32_RGB;
    out[MN_TCL_F32_ID] = MN_TC_F32_ID;
    out[MN_TCL_F32_ROWS] = MN_TC_F32_ROWS;
    out[MN_TCL_G32_SIGMA] = MN_TC_G32_SIGMA;
    out[MN_TCL_G32_RGB] = MN_TC_G32_RGB;
    out[MN_TCL_G32_ROWS] = mn_tc_g32_rows(nd.rgb_dim);
    const TcBwdWorkspace WS = tc_bwd_workspace(m, net, n_tiles128);
    out[MN_TCL_BWD_DZ] = 0;
    out[MN_TCL_BWD_GF32] = (int64_t)WS.dz_bytes;
    out[MN_TCL_BWD_EMB] = (int64_t)(WS.dz_bytes + WS.head_bytes);
    out[MN_TCL_BWD_SCALE] = (int64_t)(WS.dz_bytes + WS.head_bytes + mn_align(WS.emb_floats * sizeof(float) + 256) - 256);
    out[MN_TCL_BWD_EMB_K] = WS.emb_k;
    out[MN_TCL_BWD_HEAD_TILES] = WS.head_tiles;
    const bool layer = net.engine == TC_LAYER;
    const size_t pp0 = layer ? mn_align((size_t)WS.head_tiles * net.lin.gc * kTileM * 2) : 0;
    out[MN_TCL_BWD_DZG] = layer ? 0 : -1;
    out[MN_TCL_BWD_PP0] = layer ? (int64_t)pp0 : -1;
    out[MN_TCL_BWD_PP1] = layer ? (int64_t)(pp0 + mn_align((size_t)WS.head_tiles * net.lin.hc * kTileM * 2)) : -1;
    out[MN_TCL_N_IMG] = n_img;
    // image j of a record: trunk layer j (j < layers), F (layers), G (layers + 1); offset in the record and columns
    for (int j = 0; j < n_img; ++j) {
        out[MN_TCL_IMG + 2 * j] = (int64_t)mn_tc_img_off(j, net.lin.hc);
        out[MN_TCL_IMG + 2 * j + 1] = j == nd.layers + 1 ? net.lin.gc : net.lin.hc;
    }
    return MN_OK;
}

// Weight-gradient entry of Linear j: per input segment, the item of output channels 0..127 and the segment's first X chunk.  X is
// image j - 1 of the activation record (SRC_H) or a segment of the feature tile; dZ lies at dz_off inside a tile's gradient images.
// The output channels run in blocks of 128; a last partial block (layer engine: l.n < l.cols) reads the zero padding of the
// gradient image and stores only the channels below l.n.
static WgLinear wg_linear(const TcLinears& T, int j, int dz_off) {
    const TcLinear& l = T.l[j];
    WgLinear w{};
    for (int s = 0; s < l.nseg; ++s) {
        const TcSeg& g = l.seg[s];
        WgItem& it = w.seg[s];
        it.dz_off = dz_off;
        it.x_region = g.src == SRC_H ? 0 : 1;
        it.x_off = g.src == SRC_H ? (int)mn_tc_img_off(j - 1, T.hc) : g.src == SRC_XAUX ? (T.kpe / 8) * (kTileM * 16) : 0;
        it.n = g.k;
        it.n_real = g.k_real;
        it.m_real = l.n;
        it.w_off = l.w + g.in0;
        it.k_in = l.kin;
        it.b_off = s == 0 ? l.b : -1;      // the first segment owns the bias
        w.n_chunks[s] = (g.k + 255) / 256;
    }
    w.n_items = ((l.n + 127) / 128) * (w.n_chunks[0] + w.n_chunks[1]);
    return w;
}

int mn_train_tc_backward(mn_ctx* ctx, mn_model* m, const BwdArgs& a, int64_t n_tiles128, const TrainTcTape& tape, void* ws, size_t ws_bytes,
                         cudaStream_t st) {
    const TcNet& net = m->tc;
    if (!net.train || !m->tc_packed || !m->tc_dgrad) return mn_fail(ctx, MN_ERR_UNSUPPORTED, "tensor-core backward: unsupported network shape");
    if (n_tiles128 <= 0) return MN_OK;
    const TcBwdWorkspace WS = tc_bwd_workspace(m, net, n_tiles128);
    if (!ws || ws_bytes < WS.total) return mn_fail(ctx, MN_ERR_WORKSPACE, "mn_train_tc_backward: workspace too small");
    const NetDims& nd = a.nd;
    const TcLinears& lin = net.lin;
    const int L = nd.L, half = L / 2, hc = lin.hc;
    const int64_t act_tile = net.act_tile_bytes;
    char* wp = (char*)(((uintptr_t)ws + 255) / 256 * 256);
    unsigned char* dz = (unsigned char*)wp;               wp += WS.dz_bytes;
    float* gf32 = (float*)wp;                             wp += WS.head_bytes;
    float* emb_sum = (float*)wp;                          wp += mn_align(WS.emb_floats * sizeof(float) + 256) - 256;
    float* scale = (float*)wp;
    unsigned* maxbits = reinterpret_cast<unsigned*>(scale + 1);     // max |grad_out| (float bits), inside the same 256 bytes
    if (WS.emb_floats) MN_CUDA(ctx, cudaMemsetAsync(emb_sum, 0, WS.emb_floats * sizeof(float), st));
    MN_CUDA(ctx, cudaMemsetAsync(maxbits, 0, sizeof(unsigned), st));

    mn_prof_begin(ctx, st);   // bench.py --mode train: the whole backward of the MLP stage timed as one span
    // ---- gradient scale (power of two) from the upstream gradient
    {
        const int64_t n = a.grad_rows * a.out_cols;
        const int64_t blocks = std::min<int64_t>(std::max<int64_t>(mn_cdiv(n, (int64_t)256 * 16), 1), (int64_t)ctx->sm_count * 4);
        tc_grad_absmax_kernel<<<(unsigned)blocks, 256, 0, st>>>(a.grad_out, a.live, a.grad_rows, a.out_cols, maxbits);
        MN_LAUNCH_CHECK(ctx);
        tc_grad_scale_kernel<<<1, 32, 0, st>>>(maxbits, scale);
        MN_LAUNCH_CHECK(ctx);
    }
    MlpArgs mm{};
    mm.nd = nd;
    mm.slot_row = a.slot_row;
    mm.slot_w = a.slot_w;
    mm.counters = a.counters;
    mm.n_sub = a.n_sub;
    mm.fixed_sub = a.fixed_sub;
    mm.B = a.B;
    mm.out_cols = a.out_cols;
    mm.live = a.live;
    const int n_sub = a.counters ? a.n_sub : 1;
    // tiles the forward pass may have written: all bucketed tiles when routed, ceil(rows / 128) otherwise (the kernels stop at
    // the live rows' tiles)
    const int64_t tiles_used = a.counters ? n_tiles128 : mn_cdiv(a.B, (int64_t)kTileM);
    const int wg_smem = 2 * kWgStageBytes + 6144 + 256;
    MN_CUDA(ctx, cudaFuncSetAttribute(tc_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, wg_smem));
    // ---- sigma / rgb head weight gradients of the tiles t0 .. t0 + nt - 1, whose head-gradient blocks gf32 holds
    auto heads = [&](int64_t t0, int64_t nt) -> int {
        HeadsArgs H{};
        H.act = tape.act;
        H.gf32 = gf32;
        H.act_tile_bytes = act_tile;
        H.L = L;
        H.cols = hc;
        H.layers = nd.layers;
        H.rgb_dim = nd.rgb_dim;
        H.counters = a.counters;
        H.n_tiles = tiles_used;
        H.t_min = t0;
        H.t_max = t0 + nt;
        H.live = a.live;
        H.rows = a.B;
        H.fixed_sub = a.fixed_sub;
        H.chunk_tiles = 16;
        H.gw = a.gw;
        H.sub_stride = a.lay.total;
        H.sigma_w = a.lay.sigma_w; H.sigma_b = a.lay.sigma_b; H.rgb_w = a.lay.rgb_w; H.rgb_b = a.lay.rgb_b;
        // channel blocks: L for the sigma row; the rgb rows in groups of 16 over L/2 channels each (2 groups up to 32 rows)
        const int rgb_groups = nd.rgb_dim == 3 ? 1 : (nd.rgb_dim + 15) / 16;
        const dim3 hgrid((unsigned)mn_cdiv(nt, (int64_t)16), (unsigned)n_sub, (unsigned)mn_cdiv(std::max(L, rgb_groups * half), 256));
        if (nd.rgb_dim == 3) tc_heads_wgrad_kernel<3><<<hgrid, 256, 0, st>>>(H);
        else if (nd.rgb_dim <= MN_TC_RGB_MAX) tc_heads_wgrad_kernel<MN_TC_RGB_MAX><<<hgrid, 256, 0, st>>>(H);
        else tc_heads_wgrad_kernel<MN_TC_LG_RGB_MAX><<<hgrid, 256, 0, st>>>(H);
        MN_LAUNCH_CHECK(ctx);
        return MN_OK;
    };
    // ---- weight gradients of Linears j0 .. j1 - 1 over the tiles t0 .. t0 + nt - 1, one tc_wgrad_kernel launch.  dzt: the dZ image
    // of Linear j0 in tile t0, the tiles dz_tile_bytes apart, and the images of the later Linears after it as in a gradient record:
    // the fused engine's gradient records, or the layer engine's group buffer of its one Linear.
    auto wgrad = [&](int j0, int j1, const unsigned char* dzt, int64_t dz_tile_bytes, int64_t t0, int64_t nt) -> int {
        WgArgs W{};
        int64_t items = 0;
        for (int j = j0; j < j1; ++j) {
            W.lin[j - j0] = wg_linear(lin, j, (int)mn_tc_img_off(j - j0, hc));
            items += W.lin[j - j0].n_items;
        }
        W.act = tape.act;
        W.dz = dzt;
        W.xreg = tape.xreg;
        W.act_tile_bytes = act_tile;
        W.x_tile_bytes = net.P.x_tile_bytes;
        W.dz_tile_bytes = dz_tile_bytes;
        W.t_min = t0;
        W.t_max = t0 + nt;
        W.counters = a.counters;
        W.fixed_sub = a.fixed_sub;
        W.live = a.live;
        W.rows = a.B;
        W.gw = a.gw;
        W.sub_stride = a.lay.total;
        W.scale = scale;
        int64_t chunks;
        if (net.engine == TC_FUSED) {
            // every tile of the call, shared by n_sub sub-modules: enough CTAs to fill the machine about three times over (each
            // streams its tiles once; results are fp32 atomics)
            chunks = std::max<int64_t>(1, mn_cdiv((int64_t)ctx->sm_count * 3, items * n_sub));
            W.chunk_tiles = (int)std::max<int64_t>(8, mn_cdiv(mn_cdiv(nt, (int64_t)n_sub), chunks));
            chunks = mn_cdiv(nt, (int64_t)W.chunk_tiles);
        } else {
            // about one CTA per SM: every CTA flushes its 128 x 256 accumulators with fp32 atomics once
            chunks = std::max<int64_t>(1, mn_cdiv((int64_t)ctx->sm_count, items));
            W.chunk_tiles = (int)mn_cdiv(nt, chunks);
        }
        tc_wgrad_kernel<<<dim3((unsigned)chunks, (unsigned)items, (unsigned)n_sub), kWgThreads, wg_smem, st>>>(W);
        MN_LAUNCH_CHECK(ctx);
        return MN_OK;
    };
    int rc;

    if (net.engine == TC_FUSED) {
        // ---- data gradients: one launch of the fused kernel over the transposed images (512 wide: every GEMM in two N = 256 chunks)
        TcArgs A{};
        A.m = mm;
        A.plan = net.D;
        A.wpack = (const unsigned char*)m->tc_dgrad;
        A.n_tiles_cap = n_tiles128;
        A.tape_act = tape.act;
        A.tape_f32 = tape.f32;
        A.tape_dz = dz;
        A.tape_gf32 = gf32;
        A.grad_out = a.grad_out;
        A.emb_sum = nd.app_in_dira ? emb_sum : nullptr;
        A.scale = scale;
        A.act_tile_bytes = act_tile;
        A.layers = nd.layers;
        rc = wg_launch(ctx, A, PP_DGRAD, n_tiles128, st);
        if (rc) return rc;
        // ---- weight gradients of every Linear but rgb, straight from the gradient records.  512 wide: one launch per Linear.  A
        // single launch would be faster, but over ~80 items the chunk policy gives each CTA more tiles to sum in its accumulators,
        // which moves the gradients by more than fp32 atomic order does (DESIGN §8).
        if (L > 256) {
            for (int j = lin.n - 2; j >= 0; --j)
                if ((rc = wgrad(j, j + 1, dz + mn_tc_img_off(j, L), act_tile, 0, tiles_used))) return rc;
        } else if ((rc = wgrad(0, lin.n - 1, dz, act_tile, 0, tiles_used))) return rc;
        if ((rc = heads(0, tiles_used))) return rc;
    } else {
        // ---- layer engine, one tile group at a time: head stage -> per Linear (output side first) the weight gradient from its dZ
        // image, then the data-gradient GEMM that produces the next dZ in the other ping-pong buffer; then the sigma / rgb head
        // weight gradients.  dZ of Linear j is consumed by its weight gradient before the buffer is overwritten.
        const TcPlan& P = net.P;
        const TcPlan& D = net.D;
        const LgNet& B = net.lg;
        const int rows = mn_tc_g32_rows(nd.rgb_dim);
        const int64_t gt = WS.head_tiles;
        unsigned char* dzg = dz;                              // dZ of dir_a_encoding (gc columns)
        unsigned char* pp[2];
        pp[0] = dzg + mn_align((size_t)gt * lin.gc * kTileM * 2);
        pp[1] = pp[0] + mn_align((size_t)gt * hc * kTileM * 2);

        for (int64_t t0 = 0; t0 < tiles_used; t0 += gt) {
            const int64_t nt = tiles_used - t0 < gt ? tiles_used - t0 : gt;
            const unsigned char* rec = tape.act + t0 * act_tile;
            // ---- head stage
            {
                LdArgs H{};
                H.m = mm;
                H.tile0 = t0;
                H.grad_out = a.grad_out;
                H.tape_f32 = tape.f32;
                H.g = rec + mn_tc_img_off(nd.layers + 1, hc);
                H.g_tile_bytes = act_tile;
                H.wpack = (const unsigned char*)m->tc_packed;
                H.sub_bytes = P.sub_bytes;
                H.f32_off = P.f32_off;
                H.rgb_w_off = B.rgb_w_off;
                H.rgb_k = B.rgb_k;
                H.cols = lin.gc;
                H.gf32 = gf32;
                H.dz = dzg;
                H.emb_sum = nd.app_in_dira ? emb_sum : nullptr;
                H.scale = scale;
                if (nd.rgb_dim <= MN_TC_RGB_MAX) tc_layer_head_dgrad_kernel<MN_TC_RGB_MAX><<<(unsigned)nt, kTileM, 0, st>>>(H);
                else tc_layer_head_dgrad_kernel<MN_TC_LG_RGB_MAX><<<(unsigned)nt, kTileM, 0, st>>>(H);
                MN_LAUNCH_CHECK(ctx);
            }
            // ---- data-gradient GEMM g: dz_out = [mask](dz_in W^T) [+ S dsigma x sigma_w]
            auto dgrad = [&](unsigned char* dz_in, const TcGemm& g, unsigned char* dz_out) -> int {
                LgArgs G{};
                G.mask = g.epi != EPI_D_LINEAR ? rec + mn_tc_img_off(g.img, hc) : nullptr;     // xyz_encoding_final has no activation
                G.mask_tile_bytes = act_tile;
                G.dsig = g.epi == EPI_D_MASK_SIGMA ? gf32 + MN_TC_G32_SIGMA * kTileM : nullptr;
                G.dsig_tile_floats = (int64_t)rows * kTileM;
                G.scale = scale;
                // every column of the H-wide gradient image: the padding comes out 0 (zero weights, then the mask of a zero
                // activation), so the next GEMM and the weight gradient read whole blocks
                return lg_gemm(ctx, G, mm, D, g, m->tc_dgrad, hc, t0, nt, LgImg{}, LgImg{dz_in, (int64_t)g.k[0] * kTileM * 2, 0},
                               LgImg{dz_out, (int64_t)hc * kTileM * 2, 0}, false, true, st);
            };
            // Linear j (dir_a_encoding down to trunk layer 0): weight gradient, then data-gradient GEMM lin.n - 2 - j gives dZ of j - 1
            unsigned char* dzj = dzg;
            for (int j = lin.n - 2, nxt = 0; j >= 0; --j, nxt ^= 1) {
                if ((rc = wgrad(j, j + 1, dzj, (int64_t)lin.l[j].cols * kTileM * 2, t0, nt))) return rc;
                if (j == 0) break;
                if ((rc = dgrad(dzj, D.g[lin.n - 2 - j], pp[nxt]))) return rc;
                dzj = pp[nxt];
            }
            if ((rc = heads(t0, nt))) return rc;
        }
    }
    // ---- appearance embedding
    if (nd.app_in_dira) {
        tc_emb_grad_kernel<<<dim3((unsigned)nd.app_count, (unsigned)a.n_sub), 64, 0, st>>>(emb_sum, WS.emb_k, a.packed_bwd, a.blay.total,
                                                                                          a.blay.dira_e, half, nd.app, nd.app_count, a.gw,
                                                                                          a.lay.total, a.lay.emb);
        MN_LAUNCH_CHECK(ctx);
    }
    mn_prof_end(ctx, st);
    return MN_OK;
}
