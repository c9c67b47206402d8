// HBM-bound stages of the hot path: ray generation, depth sampling, inverse-CDF resampling,
// merge + alpha compositing, background geometry, SH head, positional encoding.
// One warp per ray for everything that scans or sorts along a ray.
//
// Arithmetic follows the oracle op for op (library compiled with -fmad=false); the two scans
// (cumprod, cumsum) accumulate in fp64 and round every prefix to fp32, which is what torch's CPU
// kernels do (SURVEY.md §8c).
#include "mn_model.cuh"

namespace {

// ------------------------------------------------------------------------------------------------
// ray generation                                                            (ray_utils.py:6-84)
// ------------------------------------------------------------------------------------------------
__global__ void ray_directions_kernel(int W, int H, float fx, float fy, float cx, float cy, int center, float* out) {
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= (int64_t)W * H) return;
    float i = (float)(p % W), j = (float)(p / W);
    if (center) { i = i + 0.5f; j = j + 0.5f; }
    const float dx = (i - cx) / fx, dy = -((j - cy) / fy), dz = -1.0f;
    const float n = sqrtf((dx * dx + dy * dy) + dz * dz);
    out[p * 3 + 0] = dx / n;
    out[p * 3 + 1] = dy / n;
    out[p * 3 + 2] = dz / n;
}

__device__ __forceinline__ bool plane_bound(const float* o, const float* d, float altitude, float* bound) {
    if (!(o[0] < altitude && d[0] > 0.0f)) return false;
    const float ndotu = -d[0];
    const float w0 = o[0] - altitude, w1 = o[1], w2 = o[2];
    const float si = w0 / ndotu;
    const float h0 = (w0 + si * d[0]) + altitude, h1 = (w1 + si * d[1]), h2 = (w2 + si * d[2]);
    const float e0 = o[0] - h0, e1 = o[1] - h1, e2 = o[2] - h2;
    *bound = sqrtf((e0 * e0 + e1 * e1) + e2 * e2);
    return true;
}

// one ray from a camera-space direction and a 3x4 pose: rotate, normalise, plane-truncated bounds (ray_utils.py:21-84)
__device__ __forceinline__ void make_ray(const float* __restrict__ dv, const float* __restrict__ M, float near, float far, int has_alt,
                                         float alt0, float alt1, float* __restrict__ r) {
    float d[3], o[3];
    for (int i = 0; i < 3; ++i) {
        float acc = dv[0] * M[i * 4 + 0];
        acc = fmaf(dv[1], M[i * 4 + 1], acc);
        acc = fmaf(dv[2], M[i * 4 + 2], acc);
        d[i] = acc;
        o[i] = M[i * 4 + 3];
    }
    const float n = sqrtf((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]);
    for (int i = 0; i < 3; ++i) d[i] = d[i] / n;
    float nb = near, fb = far;
    if (has_alt) {
        float b;
        if (plane_bound(o, d, alt0, &b)) nb = b;
        nb = fmaxf(nb, near);
        if (plane_bound(o, d, alt1, &b)) fb = b;
        fb = fminf(fb, far);
        fb = fmaxf(nb, fb);
    }
    r[0] = o[0]; r[1] = o[1]; r[2] = o[2];
    r[3] = d[0]; r[4] = d[1]; r[5] = d[2];
    r[6] = nb; r[7] = fb;
}

__global__ void rays_kernel(const float* __restrict__ dirs, int dirs_batched, const float* __restrict__ c2w, int n_poses,
                            int64_t P, float near, float far, int has_alt, float alt0, float alt1, float* out) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (int64_t)n_poses * P) return;
    const int64_t pose = t / P, p = t % P;
    make_ray(dirs + (dirs_batched ? t : p) * 3, c2w + pose * 12, near, far, has_alt, alt0, alt1, out + t * 8);
}

// The loader's use of get_rays_batch (filesystem_dataset.py:109-124) wants ONE ray per (image, pixel) pair of a chunk; the
// reference builds the full [#unique images, #unique pixels, 8] product on the device, copies it to the host and gathers the
// pairs there.  This kernel computes exactly the M pairs: ray m = (pose img_idx[m], direction pix_idx[m]).
__global__ void rays_pairs_kernel(const float* __restrict__ dirs, int64_t P, const float* __restrict__ c2w, int n_poses,
                                  const int* __restrict__ img_idx, const int* __restrict__ pix_idx, int64_t M, float near,
                                  float far, int has_alt, float alt0, float alt1, float* out, unsigned int* status) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= M) return;
    const int pose = img_idx[t], pix = pix_idx[t];
    if (pose < 0 || pose >= n_poses || pix < 0 || pix >= P) {      // the reference's fancy indexing raises IndexError here
        atomicOr(status, MN_STATUS_INDEX);
        for (int i = 0; i < 8; ++i) out[t * 8 + i] = __int_as_float(0x7fc00000);
        return;
    }
    make_ray(dirs + (int64_t)pix * 3, c2w + (int64_t)pose * 12, near, far, has_alt, alt0, alt1, out + t * 8);
}

// ------------------------------------------------------------------------------------------------
// training batch assembly                      (DataLoader over FilesystemDataset / MemoryDataset)
// ------------------------------------------------------------------------------------------------
// Up to three row-major columns of 4-byte elements gathered at the rows of an index slice: out[b] = src[idx[b]].  A column is
// moved in 16-byte units where its row width is a multiple of 4 elements and both pointers are 16-byte aligned, else element
// by element.  One thread per (batch row, unit); the units of the three columns are laid end to end.
struct GatherArgs {
    const unsigned int* src[3];
    unsigned int* dst[3];
    int w[3];        // row width in 4-byte elements (0: no column)
    int vec[3];      // 1: 16-byte units
    int units[3];    // units per row
    int row_units;   // units[0] + units[1] + units[2]
};

// v[c] with c in 0..2 by selects, so that the kernel parameters are not copied to local memory for a dynamic index
template <class T>
__device__ __forceinline__ T pick3(const T (&v)[3], int c) { return c == 0 ? v[0] : (c == 1 ? v[1] : v[2]); }

__global__ void gather_batch_kernel(const int64_t* __restrict__ idx, int64_t B, int64_t n_rows, const GatherArgs a,
                                    unsigned int* status) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= B * a.row_units) return;
    const int64_t b = t / a.row_units;
    const int first = (int)(t % a.row_units);
    int u = first, c = 0;
    if (u >= a.units[0]) {
        u -= a.units[0];
        c = 1;
        if (u >= a.units[1]) { u -= a.units[1]; c = 2; }
    }
    const unsigned int* src = pick3(a.src, c);
    unsigned int* dst = pick3(a.dst, c);
    const int w = pick3(a.w, c);
    const int64_t row = idx[b];
    const bool ok = row >= 0 && row < n_rows;
    if (!ok && first == 0) atomicOr(status, MN_STATUS_INDEX);    // the reference's tensor indexing raises IndexError
    if (pick3(a.vec, c)) {
        uint4* d = reinterpret_cast<uint4*>(dst + b * w) + u;
        *d = ok ? __ldg(reinterpret_cast<const uint4*>(src + row * w) + u) : make_uint4(~0u, ~0u, ~0u, ~0u);
    } else {
        dst[b * w + u] = ok ? __ldg(src + row * w + u) : ~0u;
    }
}

// ------------------------------------------------------------------------------------------------
// depth sampling                                               (rendering.py:82-87, 472-483)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float lerp_depth(float near, float far, float t) { return near * (1.0f - t) + far * t; }

__global__ void sample_coarse_kernel(const float* __restrict__ rays, const float* __restrict__ far_ov,
                                     const float* __restrict__ steps, const float* __restrict__ rnd, float perturb,
                                     int64_t N, int S, float* __restrict__ z_out, float* __restrict__ xyz_out) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= N * S) return;
    const int64_t ray = t / S;
    const int s = (int)(t % S);
    const float* r = rays + ray * 8;
    const float near = r[6], far = far_ov ? far_ov[ray] : r[7];
    float z = lerp_depth(near, far, steps[s]);
    if (perturb > 0.0f) {
        const float lower = s > 0 ? 0.5f * (lerp_depth(near, far, steps[s - 1]) + z) : z;
        const float upper = s < S - 1 ? 0.5f * (z + lerp_depth(near, far, steps[s + 1])) : z;
        z = lower + (upper - lower) * (perturb * rnd[t]);
    }
    z_out[t] = z;
    if (xyz_out) {
        xyz_out[t * 3 + 0] = r[0] + r[3] * z;
        xyz_out[t * 3 + 1] = r[1] + r[4] * z;
        xyz_out[t * 3 + 2] = r[2] + r[5] * z;
    }
}

// flip (perturb == 0 only): row written in reverse order, torch.flip(z, [-1])
__global__ void stratify_kernel(const float* __restrict__ zin, int64_t stride, const float* __restrict__ rnd, float perturb,
                                int64_t N, int S, float* __restrict__ z_out, LiveRows live, int flip) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= live.rows(N) * S) return;
    const int64_t ray = t / S;
    const int s = (int)(t % S);
    const float* zr = zin + ray * stride;
    float z = zr[flip ? S - 1 - s : s];
    if (perturb > 0.0f) {
        const float lower = s > 0 ? 0.5f * (zr[s - 1] + z) : z;
        const float upper = s < S - 1 ? 0.5f * (z + zr[s + 1]) : z;
        z = lower + (upper - lower) * (perturb * rnd[t]);
    }
    z_out[t] = z;
}

__global__ void points_from_z_kernel(const float* __restrict__ rays, const float* __restrict__ z, int64_t N, int S,
                                     float* __restrict__ xyz) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= N * S) return;
    const float* r = rays + (t / S) * 8;
    const float zz = z[t];
    xyz[t * 3 + 0] = r[0] + r[3] * zz;
    xyz[t * 3 + 1] = r[1] + r[4] * zz;
    xyz[t * 3 + 2] = r[2] + r[5] * zz;
}

// ------------------------------------------------------------------------------------------------
// warp-level helpers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ double warp_incl_scan_mul(double v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const double u = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v = v * u;
    }
    return v;
}
__device__ __forceinline__ double warp_incl_scan_add(double v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const double u = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v = v + u;
    }
    return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// bitonic sort of n (power of two) (key, id) pairs held in shared memory by one warp; total order is
// (key, id) so equal depths keep a deterministic order.
__device__ __forceinline__ void warp_bitonic(float* key, unsigned short* id, int n, bool descending, int lane) {
    for (int k = 2; k <= n; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = lane; i < n; i += 32) {
                const int l = i ^ j;
                if (l > i) {
                    const float a = key[i], b = key[l];
                    const unsigned short ia = id[i], ib = id[l];
                    bool gt = (a > b) || (a == b && ia > ib);     // element i sorts after element l (ascending)
                    if (descending) gt = (a < b) || (a == b && ia > ib);
                    const bool up = ((i & k) == 0);
                    if (gt == up) {
                        key[i] = b; key[l] = a;
                        id[i] = ib; id[l] = ia;
                    }
                }
            }
            __syncwarp();
        }
    }
}

// ------------------------------------------------------------------------------------------------
// merge + composite                                                   (rendering.py:336-393)
// ------------------------------------------------------------------------------------------------
// Shared memory of one warp (one ray) of the composite kernels, 4 warps per CTA: the float planes [4 warps][2][npad]
// come first, then the id planes [2][4 warps][npad]; the second id plane (merge scratch, at ids + 4 npad) is only
// addressed inside composite_merge.
struct CompositeSmem {
    float* zs;             // merged depths
    float* f2;             // merge scratch, then a per-sample float of the kernel
    unsigned short* ids;   // sample index of each merged position (< S: own sample, else stored sample + S)
};
__device__ __forceinline__ CompositeSmem composite_smem(unsigned char* sm_raw, int warp, int npad) {
    CompositeSmem s;
    s.zs = reinterpret_cast<float*>(sm_raw) + (size_t)warp * npad * 2;
    s.f2 = s.zs + npad;
    s.ids = reinterpret_cast<unsigned short*>(reinterpret_cast<float*>(sm_raw) + (size_t)4 * npad * 2) + (size_t)warp * npad;
    return s;
}

int pow2_at_least(int v) {
    int p = 32;
    while (p < v) p <<= 1;
    return p;
}

// Launches either composite kernel: one warp per ray, 4 rays per CTA, each warp with the buffers of composite_smem.
template <class Args>
int composite_launch(mn_ctx* ctx, void (*kernel)(Args), Args a, const char* name, cudaStream_t st) {
    a.npad = a.S2 > 0 ? pow2_at_least(a.S + a.S2) : (a.S + 31) / 32 * 32;
    if (a.npad > 4096) return mn_fail(ctx, MN_ERR_UNSUPPORTED, std::string(name) + ": more than 4096 samples per ray");
    const size_t sm = (size_t)4 * a.npad * (2 * sizeof(float) + 2 * sizeof(unsigned short));
    MN_CUDA(ctx, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
    kernel<<<(unsigned)mn_cdiv(a.N, 4), 128, sm, st>>>(a);
    MN_LAUNCH_CHECK(ctx);
    return MN_OK;
}

// Loads the ray's own depths and the stored ones into s.zs / s.ids in merged order: (depth, index), own samples first on
// ties.  The backward pass is only right because it rebuilds exactly this order.  Returns the max over the own depths (the
// last-delta fix-up).  Args: CompositeArgs or CompositeBwdArgs.
template <class Args>
__device__ __forceinline__ float composite_merge(const Args& a, int64_t ray, int lane, const CompositeSmem& s) {
    float* zs = s.zs;
    unsigned short* ids = s.ids;
    const int n = a.S + a.S2;
    float zmax = -INFINITY;
    for (int i = lane; i < a.S; i += 32) {
        const float v = a.z[ray * a.S + i];
        zs[i] = v;
        ids[i] = (unsigned short)i;
        zmax = fmaxf(zmax, v);
    }
    zmax = warp_max(zmax);
    if (a.S2 > 0) {
        for (int i = lane; i < a.S2; i += 32) {
            zs[a.S + i] = a.z2[ray * a.S2 + i];
            ids[a.S + i] = (unsigned short)(a.S + i);
        }
        __syncwarp();
        // Both runs are usually already ordered (deterministic sampling): merge by rank instead of sorting.
        // Same total order as the bitonic path.
        bool ordered = true;
        for (int i = lane; i + 1 < a.S; i += 32) ordered &= a.flip ? (zs[i] >= zs[i + 1]) : (zs[i] <= zs[i + 1]);
        for (int i = lane; i + 1 < a.S2; i += 32)
            ordered &= a.flip ? (zs[a.S + i] >= zs[a.S + i + 1]) : (zs[a.S + i] <= zs[a.S + i + 1]);
        ordered = __all_sync(0xffffffffu, ordered);
        if (ordered) {
            float* zm = s.f2;
            unsigned short* idm = ids + a.npad * 4;
            for (int i = lane; i < n; i += 32) {
                const bool own = i < a.S;
                const float v = zs[i];
                const float* other = own ? zs + a.S : zs;
                const int m = own ? a.S2 : a.S;
                // own element: count others strictly before it; other element: count own elements before-or-equal
                int lo = 0, hi = m;
                while (lo < hi) {
                    const int mid = (lo + hi) >> 1;
                    const float o = other[mid];
                    const bool before = a.flip ? (own ? o > v : o >= v) : (own ? o < v : o <= v);
                    if (before) lo = mid + 1; else hi = mid;
                }
                const int pos = (own ? i : i - a.S) + lo;
                zm[pos] = v;
                idm[pos] = (unsigned short)i;
            }
            __syncwarp();
            for (int i = lane; i < n; i += 32) { const float v = zm[i]; const unsigned short id = idm[i]; zs[i] = v; ids[i] = id; }
        } else {
            const float pad = a.flip ? -INFINITY : INFINITY;
            for (int i = n + lane; i < a.npad; i += 32) { zs[i] = pad; ids[i] = 0xFFFF; }
            __syncwarp();
            warp_bitonic(zs, ids, a.npad, a.flip != 0, lane);
        }
    }
    __syncwarp();
    return zmax;
}

// Distance from merged sample p to the next one; the last sample takes the ray's last delta ld.
__device__ __forceinline__ float sample_delta(const float* zs, int p, int n, int flip, float ld) {
    const float zz = zs[p];
    const float znext = (p + 1 < n) ? zs[p + 1] : 0.0f;
    float delta = flip ? (zz - znext) : (znext - zz);
    if (p + 1 == n) delta = ld;
    return delta;
}

struct CompositeArgs {
    const float* raw;      // [N,S,4]
    const float* z;        // [N,S]
    const float* dreal;    // [N,S] or null
    int S;
    const float* raw2;     // [N,S2,4] or null
    const float* z2;
    const float* dreal2;
    int S2;
    const float* last_delta;  // [N]
    int64_t N;
    int flip;
    float *weights, *rgb, *depth, *var, *lambda;
    int npad;              // shared-memory elements per warp
    LiveRows live;         // rays at or past live.rows(N) are skipped
};

__global__ void __launch_bounds__(128) composite_kernel(const CompositeArgs a) {
    extern __shared__ unsigned char sm_raw[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t ray = (int64_t)blockIdx.x * 4 + warp;
    if (ray >= a.live.rows(a.N)) return;
    const int n = a.S + a.S2;
    const CompositeSmem sm = composite_smem(sm_raw, warp, a.npad);
    const float* zs = sm.zs;
    float* ws = sm.f2;
    const unsigned short* ids = sm.ids;
    const float zmax = composite_merge(a, ray, lane, sm);

    float ld = a.last_delta[ray];
    if (ld < 1e10f) ld = ld - zmax;   // rendering.py:191-193 / 224-225: max over this pass's own depths

    double carry = 1.0;        // running fp64 product
    float carry_f = 1.0f;      // its fp32 rounding == T of the previous sample
    double acc_r = 0, acc_g = 0, acc_b = 0, acc_d = 0;
    for (int c0 = 0; c0 < n; c0 += 32) {
        const int p = c0 + lane;
        const bool ok = p < n;
        float alpha = 0.0f, x = 1.0f, cr = 0, cg = 0, cb = 0, zz = 0, dd = 0;
        if (ok) {
            const int id = ids[p];
            const float* rw = (id < a.S) ? a.raw + (ray * a.S + id) * 4 : a.raw2 + (ray * a.S2 + (id - a.S)) * 4;
            const float4 v = *reinterpret_cast<const float4*>(rw);
            cr = v.x; cg = v.y; cb = v.z;
            zz = zs[p];
            const float delta = sample_delta(zs, p, n, a.flip, ld);
            alpha = 1.0f - expf(-delta * v.w);
            x = (1.0f - alpha) + 1e-8f;
            dd = zz;
            if (a.dreal) dd = (id < a.S) ? a.dreal[ray * a.S + id] : a.dreal2[ray * a.S2 + (id - a.S)];
        }
        const double incl = warp_incl_scan_mul((double)x, lane);
        const double Pd = carry * incl;
        const float Tf = (float)Pd;
        float Tprev = __shfl_up_sync(0xffffffffu, Tf, 1);
        if (lane == 0) Tprev = carry_f;
        const float w = alpha * Tprev;
        if (ok) {
            ws[p] = w;
            acc_r += (double)(w * cr);
            acc_g += (double)(w * cg);
            acc_b += (double)(w * cb);
            acc_d += (double)(w * dd);
        }
        const int last = min(31, n - 1 - c0);
        carry = __shfl_sync(0xffffffffu, Pd, last);
        carry_f = __shfl_sync(0xffffffffu, Tf, last);
    }
    acc_r = warp_sum(acc_r); acc_g = warp_sum(acc_g); acc_b = warp_sum(acc_b); acc_d = warp_sum(acc_d);
    const float depth = (float)acc_d;
    __syncwarp();
    if (a.var) {
        double acc_v = 0;
        for (int p = lane; p < n; p += 32) {
            const float t = zs[p] - depth;
            acc_v += (double)(ws[p] * (t * t));
        }
        acc_v = warp_sum(acc_v);
        if (lane == 0) a.var[ray] = (float)acc_v;
    }
    if (a.weights)
        for (int p = lane; p < n; p += 32) a.weights[ray * n + p] = ws[p];
    if (lane == 0) {
        if (a.rgb) { a.rgb[ray * 3 + 0] = (float)acc_r; a.rgb[ray * 3 + 1] = (float)acc_g; a.rgb[ray * 3 + 2] = (float)acc_b; }
        if (a.depth) a.depth[ray] = depth;
        if (a.lambda) a.lambda[ray] = carry_f;
    }
}

// ------------------------------------------------------------------------------------------------
// inverse-CDF resampling                                              (rendering.py:486-536)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) sample_pdf_kernel(const float* __restrict__ zc, const float* __restrict__ weights,
                                                         int64_t w_stride, const float* __restrict__ cdf_in,
                                                         const float* __restrict__ u, int64_t u_stride, int64_t N, int S,
                                                         int F, float* __restrict__ z_out, int64_t* __restrict__ inds_out,
                                                         float* __restrict__ cdf_out, LiveRows live) {
    extern __shared__ unsigned char sm_raw[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t ray = (int64_t)blockIdx.x * 4 + warp;
    if (ray >= live.rows(N)) return;
    const int nb = S - 2;          // pdf / cdf entries
    const int nc = S - 1;          // padded cdf entries == number of bin edges
    float* cs = reinterpret_cast<float*>(sm_raw) + (size_t)warp * 2 * S;
    float* bins = cs + S;
    for (int i = lane; i < nc; i += 32) bins[i] = 0.5f * (zc[ray * S + i] + zc[ray * S + i + 1]);   // :213
    if (cdf_in) {
        for (int i = lane; i < nb; i += 32) cs[i + 1] = cdf_in[ray * nb + i];
        if (lane == 0) cs[0] = 0.0f;
    } else {
        const float* wr = weights + ray * w_stride + 1;     // weights_coarse[:, 1:-1]
        double tot = 0.0;
        for (int i = lane; i < nb; i += 32) tot += (double)(wr[i] + 1e-8f);
        const float sum = (float)warp_sum(tot);
        double carry = 0.0;
        for (int c0 = 0; c0 < nb; c0 += 32) {
            const int i = c0 + lane;
            const float pdf = (i < nb) ? (wr[i] + 1e-8f) / sum : 0.0f;
            const double incl = carry + warp_incl_scan_add((double)pdf, lane);
            if (i < nb) cs[i + 1] = (float)incl;
            carry = __shfl_sync(0xffffffffu, incl, 31);
        }
        if (lane == 0) cs[0] = 0.0f;
    }
    __syncwarp();
    if (cdf_out)
        for (int i = lane; i < nb; i += 32) cdf_out[ray * nb + i] = cs[i + 1];
    for (int j = lane; j < F; j += 32) {
        const float uu = u[ray * u_stride + j];
        int lo = 0, hi = nc;   // first index with cs[idx] > uu   (searchsorted right=True)
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (cs[mid] <= uu) lo = mid + 1; else hi = mid;
        }
        const int inds = lo;
        const int below = max(inds - 1, 0), above = min(inds, nb);
        const float cb = cs[below], ca = cs[above];
        float denom = ca - cb;
        if (denom < 1e-8f) denom = 1.0f;
        const float bb = bins[below], ba = bins[above];
        z_out[ray * F + j] = bb + ((uu - cb) / denom) * (ba - bb);
        if (inds_out) inds_out[ray * F + j] = inds;
    }
}

// out_flip (optional): the same rows in reverse order, torch.flip(out, [-1])
__global__ void __launch_bounds__(128) sort_cat_kernel(const float* __restrict__ a, int na, const float* __restrict__ b,
                                                       int nb, int64_t N, int descending, int npad,
                                                       float* __restrict__ out, float* __restrict__ out_flip, LiveRows live) {
    extern __shared__ unsigned char sm_raw[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t ray = (int64_t)blockIdx.x * 4 + warp;
    if (ray >= live.rows(N)) return;
    float* key = reinterpret_cast<float*>(sm_raw) + (size_t)warp * npad;
    unsigned short* id = reinterpret_cast<unsigned short*>(reinterpret_cast<float*>(sm_raw) + (size_t)4 * npad) +
                         (size_t)warp * npad;
    const int n = na + nb;
    for (int i = lane; i < na; i += 32) { key[i] = a[ray * na + i]; id[i] = (unsigned short)i; }
    for (int i = lane; i < nb; i += 32) { key[na + i] = b[ray * nb + i]; id[na + i] = (unsigned short)(na + i); }
    const float pad = descending ? -INFINITY : INFINITY;
    for (int i = n + lane; i < npad; i += 32) { key[i] = pad; id[i] = 0xFFFF; }
    __syncwarp();
    warp_bitonic(key, id, npad, descending != 0, lane);
    for (int i = lane; i < n; i += 32) out[ray * n + i] = key[i];
    if (out_flip)
        for (int i = lane; i < n; i += 32) out_flip[ray * n + (n - 1 - i)] = key[i];
}

// ------------------------------------------------------------------------------------------------
// background geometry                                                  (rendering.py:396-469)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float dot3(const float* a, const float* b) { return mn_dot3(a, b); }

__global__ void intersect_sphere_kernel(const float* __restrict__ rays, const float* __restrict__ center,
                                        const float* __restrict__ radius, int64_t N, float* __restrict__ fg_far,
                                        unsigned int* status) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    bool outside;
    fg_far[i] = mn_sphere_far(rays + i * 8, center, radius, &outside);
    if (outside) atomicOr(status, MN_STATUS_SPHERE);
}

// flip_pts: the points of each ray are written in reverse sample order (torch.flip(pts, [-2])), depth_real in sample order
__global__ void points_outside_kernel(const float* __restrict__ rays, const int64_t* __restrict__ ids,
                                      const float* __restrict__ depth, const float* __restrict__ center,
                                      const float* __restrict__ radius, int64_t n, int S, int real, int c2d,
                                      float* __restrict__ pts, float* __restrict__ depth_real, LiveRows live, int flip_pts) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= live.rows(n) * S) return;
    const int64_t r = t / S;
    const int64_t ray = ids ? ids[r] : r;
    float o0[3], d0[3], o[3], d[3];
    for (int j = 0; j < 3; ++j) {
        o0[j] = rays[ray * 8 + j];
        d0[j] = rays[ray * 8 + 3 + j];
        o[j] = o0[j]; d[j] = d0[j];
        if (radius) { o[j] = (o[j] - center[j]) / radius[j]; d[j] = d[j] / radius[j]; }
    }
    const float dd = dot3(d, d);
    const float d1 = -dot3(d, o) / dd;
    float pm[3];
    for (int j = 0; j < 3; ++j) pm[j] = o[j] + d1 * d[j];
    const float pmn = sqrtf(dot3(pm, pm));
    const float cosv = 1.0f / sqrtf(dd);
    const float d2 = sqrtf(1.0f - pmn * pmn) * cosv;
    float ps[3];
    for (int j = 0; j < 3; ++j) ps[j] = o[j] + (d1 + d2) * d[j];
    float ax[3] = {o[1] * ps[2] - o[2] * ps[1], o[2] * ps[0] - o[0] * ps[2], o[0] * ps[1] - o[1] * ps[0]};
    const float an = sqrtf(dot3(ax, ax)) + 1e-8f;
    for (int j = 0; j < 3; ++j) ax[j] = ax[j] / an;
    const float dep = depth[t];
    const float phi = asinf(pmn);
    const float theta = asinf(pmn * dep);
    const float ang = phi - theta;
    const float ca = cosf(ang), sa = sinf(ang);
    const float cr[3] = {ax[1] * ps[2] - ax[2] * ps[1], ax[2] * ps[0] - ax[0] * ps[2], ax[0] * ps[1] - ax[1] * ps[0]};
    const float adp = dot3(ax, ps);
    float pn[3];
    for (int j = 0; j < 3; ++j) pn[j] = (ps[j] * ca + cr[j] * sa) + (ax[j] * adp) * (1.0f - ca);
    const float nn = sqrtf(dot3(pn, pn));
    for (int j = 0; j < 3; ++j) pn[j] = pn[j] / nn;
    const float dr = (1.0f / (dep + 1e-8f)) * cosf(theta) + d1;
    depth_real[t] = dr;
    const int C = real ? 7 : 4;
    float* q = pts + (flip_pts ? r * S + (S - 1 - (t - r * S)) : t) * C;
    if (real) {
        const float s = c2d ? dr : (d1 + d2);
        for (int j = 0; j < 3; ++j) q[j] = o0[j] + d0[j] * s;
        q += 3;
    }
    q[0] = pn[0]; q[1] = pn[1]; q[2] = pn[2]; q[3] = dep;
}

// ------------------------------------------------------------------------------------------------
// SH head + sigmoid                               (spherical_harmonics.py:55-106, rendering.py:301-306)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float sh_eval(int deg, const float* s, float x, float y, float z) {
    const float C0 = 0.28209479177387814f, C1 = 0.4886025119029199f;
    float r = C0 * s[0];
    if (deg < 1) return r;
    r = ((r - (C1 * y) * s[1]) + (C1 * z) * s[2]) - (C1 * x) * s[3];
    if (deg < 2) return r;
    const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
    r = ((((r + (1.0925484305920792f * xy) * s[4]) + (-1.0925484305920792f * yz) * s[5]) +
          (0.31539156525252005f * ((2.0f * zz - xx) - yy)) * s[6]) + (-1.0925484305920792f * xz) * s[7]) +
        (0.5462742152960396f * (xx - yy)) * s[8];
    if (deg < 3) return r;
    r = ((((((r + ((-0.5900435899266435f * y) * (3 * xx - yy)) * s[9]) + ((2.890611442640554f * xy) * z) * s[10]) +
            ((-0.4570457994644658f * y) * ((4 * zz - xx) - yy)) * s[11]) +
           ((0.3731763325901154f * z) * ((2 * zz - 3 * xx) - 3 * yy)) * s[12]) +
          ((-0.4570457994644658f * x) * ((4 * zz - xx) - yy)) * s[13]) + ((1.445305721320277f * z) * (xx - yy)) * s[14]) +
        ((-0.5900435899266435f * x) * (xx - 3 * yy)) * s[15];
    if (deg < 4) return r;
    r = ((((((((r + ((2.5033429417967046f * xy) * (xx - yy)) * s[16]) + ((-1.7701307697799304f * yz) * (3 * xx - yy)) * s[17]) +
              ((0.9461746957575601f * xy) * (7 * zz - 1)) * s[18]) + ((-0.6690465435572892f * yz) * (7 * zz - 3)) * s[19]) +
            (0.10578554691520431f * (zz * (35 * zz - 30) + 3)) * s[20]) + ((-0.6690465435572892f * xz) * (7 * zz - 3)) * s[21]) +
          ((0.47308734787878004f * (xx - yy)) * (7 * zz - 1)) * s[22]) + ((-1.7701307697799304f * xz) * (xx - 3 * yy)) * s[23]) +
        (0.6258357354491761f * (xx * (xx - 3 * yy) - yy * (3 * xx - yy))) * s[24];
    return r;
}

__global__ void sh_to_rgb_kernel(int deg, const float* __restrict__ coef, int64_t cstride, const float* __restrict__ dirs,
                                 int64_t dstride, int ddiv, int64_t B, int sig, float* __restrict__ out, LiveRows live,
                                 const int* __restrict__ gather) {
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= live.rows(B)) return;
    const int nc = (deg + 1) * (deg + 1);
    const float* c = coef + b * cstride;
    // gather: row b is the compacted sample gather[b] (an occupancy-grid query), whose ray gives the direction
    const float* d = dirs + ((gather ? (int64_t)gather[b] : b) / ddiv) * dstride;
    float s[25];
    float o[4];
    for (int ch = 0; ch < 3; ++ch) {
        for (int k = 0; k < nc; ++k) s[k] = c[ch * nc + k];
        const float v = sh_eval(deg, s, d[0], d[1], d[2]);
        o[ch] = sig ? mn_sigmoid(v) : v;
    }
    o[3] = c[3 * nc];
    *reinterpret_cast<float4*>(out + b * 4) = make_float4(o[0], o[1], o[2], o[3]);
}

__global__ void embed_kernel(const float* __restrict__ x, int64_t B, int dim, int nf, float* __restrict__ out) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int per = dim * (1 + nf);
    if (t >= B * per) return;
    const int64_t b = t / per;
    const int q = (int)(t % per);
    const int width = dim * (1 + 2 * nf);
    float* o = out + b * width;
    if (q < dim) {
        o[q] = x[b * dim + q];
    } else {
        const int qq = q - dim, k = qq / dim, j = qq % dim;
        float s, c;
        mn_pe_sincos(x[b * dim + j], k, &s, &c);
        o[dim + k * 2 * dim + j] = s;
        o[dim + k * 2 * dim + dim + j] = c;
    }
}


// ------------------------------------------------------------------------------------------------
// backward of merge + composite                       (rendering.py:336-373; SURVEY.md §8f-1)
// ------------------------------------------------------------------------------------------------
// With x_j = 1 - alpha_j + 1e-8, T_j = prod_{k<j} x_k, w_j = alpha_j T_j, rgb = sum_j w_j c_j,
// lambda = prod_j x_j and upstream gradients g (rgb) and gl (lambda):
//     dL/dc_j     = w_j g
//     dL/dalpha_j = T_j (g.c_j) - ( sum_{i>j} w_i (g.c_i) + lambda gl ) / x_j
//     dL/dsigma_j = dL/dalpha_j * delta_j * exp(-delta_j sigma_j)
// The merged order is rebuilt exactly like composite_kernel does (same total order on ties), T comes from
// the same fp64 prefix product rounded to fp32, the suffix sum runs in fp64.
struct CompositeBwdArgs {
    const float* raw; const float* z; int S;
    const float* raw2; const float* z2; int S2;
    const float* last_delta;
    int64_t N;
    int flip;
    const float* grad_rgb;      // [N,3]
    const float* grad_lambda;   // [N] or null
    float* grad_raw;            // [N,S,4]
    float* grad_raw2;           // [N,S2,4]
    int npad;
    LiveRows live;              // rays at or past live.rows(N) are skipped
};

__device__ __forceinline__ double warp_incl_suffix_add(double v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const double u = __shfl_down_sync(0xffffffffu, v, o);
        if (lane + o < 32) v = v + u;
    }
    return v;
}

__global__ void __launch_bounds__(128) composite_bwd_kernel(const CompositeBwdArgs a) {
    extern __shared__ unsigned char sm_raw[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t ray = (int64_t)blockIdx.x * 4 + warp;
    if (ray >= a.live.rows(a.N)) return;
    const int n = a.S + a.S2;
    const CompositeSmem sm = composite_smem(sm_raw, warp, a.npad);
    const float* zs = sm.zs;
    float* ts = sm.f2;   // T (exclusive transmittance) per merged position
    const unsigned short* ids = sm.ids;
    const float zmax = composite_merge(a, ray, lane, sm);

    float ld = a.last_delta[ray];
    if (ld < 1e10f) ld = ld - zmax;

    // forward sweep: exclusive transmittance T (fp32-rounded fp64 prefix product, as composite_kernel)
    double carry = 1.0;
    float carry_f = 1.0f;
    for (int c0 = 0; c0 < n; c0 += 32) {
        const int p = c0 + lane;
        const bool ok = p < n;
        float x = 1.0f;
        if (ok) {
            const int id = ids[p];
            const float sg = (id < a.S) ? a.raw[(ray * a.S + id) * 4 + 3] : a.raw2[(ray * a.S2 + (id - a.S)) * 4 + 3];
            const float delta = sample_delta(zs, p, n, a.flip, ld);
            const float alpha = 1.0f - expf(-delta * sg);
            x = (1.0f - alpha) + 1e-8f;
        }
        const double incl = warp_incl_scan_mul((double)x, lane);
        const double Pd = carry * incl;
        const float Tf = (float)Pd;
        float Tprev = __shfl_up_sync(0xffffffffu, Tf, 1);
        if (lane == 0) Tprev = carry_f;
        if (ok) ts[p] = Tprev;
        const int last = min(31, n - 1 - c0);
        carry = __shfl_sync(0xffffffffu, Pd, last);
        carry_f = __shfl_sync(0xffffffffu, Tf, last);
    }
    __syncwarp();
    const float g0 = a.grad_rgb[ray * 3 + 0], g1 = a.grad_rgb[ray * 3 + 1], g2 = a.grad_rgb[ray * 3 + 2];
    const double lam_term = a.grad_lambda ? (double)carry_f * (double)a.grad_lambda[ray] : 0.0;

    // backward sweep, last chunk first
    double tail = 0.0;   // sum of w_i (g.c_i) over all later chunks
    for (int c0 = ((n - 1) / 32) * 32; c0 >= 0; c0 -= 32) {
        const int p = c0 + lane;
        const bool ok = p < n;
        double wG = 0.0, G = 0.0;
        float w = 0.0f, x = 1.0f, delta = 0.0f, ex = 0.0f, Tp = 0.0f;
        int id = 0;
        if (ok) {
            id = ids[p];
            const float* rw = (id < a.S) ? a.raw + (ray * a.S + id) * 4 : a.raw2 + (ray * a.S2 + (id - a.S)) * 4;
            const float4 v = *reinterpret_cast<const float4*>(rw);
            delta = sample_delta(zs, p, n, a.flip, ld);
            ex = expf(-delta * v.w);
            const float alpha = 1.0f - ex;
            x = (1.0f - alpha) + 1e-8f;
            Tp = ts[p];
            w = alpha * Tp;
            G = (double)g0 * (double)v.x + (double)g1 * (double)v.y + (double)g2 * (double)v.z;
            wG = (double)w * G;
        }
        const double sfx = warp_incl_suffix_add(wG, lane);          // sum over lanes >= this one
        const double later = (sfx - wG) + tail;                      // strictly later samples
        if (ok) {
            const double d_alpha = (double)Tp * G - (later + lam_term) / (double)x;
            const float d_sigma = (float)(d_alpha * (double)delta * (double)ex);
            float* out = (id < a.S) ? a.grad_raw + (ray * a.S + id) * 4 : a.grad_raw2 + (ray * a.S2 + (id - a.S)) * 4;
            *reinterpret_cast<float4*>(out) = make_float4(w * g0, w * g1, w * g2, d_sigma);
        }
        tail += __shfl_sync(0xffffffffu, sfx, 0);
    }
}

// Real SH basis values with the constants folded in: sh_eval(deg, s, d) == sum_k Y[k] * s[k].
__device__ __forceinline__ void sh_basis(int deg, float x, float y, float z, float* Y) {
    Y[0] = 0.28209479177387814f;
    if (deg < 1) return;
    const float C1 = 0.4886025119029199f;
    Y[1] = -(C1 * y); Y[2] = C1 * z; Y[3] = -(C1 * x);
    if (deg < 2) return;
    const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
    Y[4] = 1.0925484305920792f * xy;
    Y[5] = -1.0925484305920792f * yz;
    Y[6] = 0.31539156525252005f * ((2.0f * zz - xx) - yy);
    Y[7] = -1.0925484305920792f * xz;
    Y[8] = 0.5462742152960396f * (xx - yy);
    if (deg < 3) return;
    Y[9] = (-0.5900435899266435f * y) * (3 * xx - yy);
    Y[10] = (2.890611442640554f * xy) * z;
    Y[11] = (-0.4570457994644658f * y) * ((4 * zz - xx) - yy);
    Y[12] = (0.3731763325901154f * z) * ((2 * zz - 3 * xx) - 3 * yy);
    Y[13] = (-0.4570457994644658f * x) * ((4 * zz - xx) - yy);
    Y[14] = (1.445305721320277f * z) * (xx - yy);
    Y[15] = (-0.5900435899266435f * x) * (xx - 3 * yy);
    if (deg < 4) return;
    Y[16] = (2.5033429417967046f * xy) * (xx - yy);
    Y[17] = (-1.7701307697799304f * yz) * (3 * xx - yy);
    Y[18] = (0.9461746957575601f * xy) * (7 * zz - 1);
    Y[19] = (-0.6690465435572892f * yz) * (7 * zz - 3);
    Y[20] = 0.10578554691520431f * (zz * (35 * zz - 30) + 3);
    Y[21] = (-0.6690465435572892f * xz) * (7 * zz - 3);
    Y[22] = (0.47308734787878004f * (xx - yy)) * (7 * zz - 1);
    Y[23] = (-1.7701307697799304f * xz) * (xx - 3 * yy);
    Y[24] = 0.6258357354491761f * (xx * (xx - 3 * yy) - yy * (3 * xx - yy));
}

__global__ void sh_to_rgb_bwd_kernel(int deg, const float* __restrict__ coef, int64_t cstride, const float* __restrict__ dirs,
                                     int64_t dstride, int ddiv, int64_t B, int sig, const float* __restrict__ gout,
                                     float* __restrict__ gcoef, LiveRows live, const int* __restrict__ gather) {
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= live.rows(B)) return;
    const int nc = (deg + 1) * (deg + 1);
    const float* c = coef + b * cstride;
    const float* d = dirs + ((gather ? (int64_t)gather[b] : b) / ddiv) * dstride;     // as sh_to_rgb_kernel
    float* gc = gcoef + b * cstride;
    float Y[25], s[25];
    sh_basis(deg, d[0], d[1], d[2], Y);
    for (int ch = 0; ch < 3; ++ch) {
        float g = gout[b * 4 + ch];
        if (sig) {
            for (int k = 0; k < nc; ++k) s[k] = c[ch * nc + k];
            const float o = mn_sigmoid(sh_eval(deg, s, d[0], d[1], d[2]));
            g = (g * (1.0f - o)) * o;
        }
        for (int k = 0; k < nc; ++k) gc[ch * nc + k] = g * Y[k];
    }
    gc[3 * nc] = gout[b * 4 + 3];
}

}  // namespace

// =================================================================================================
extern "C" {

int mn_ray_directions(mn_ctx* ctx, int W, int H, float fx, float fy, float cx, float cy, int center_pixels, float* out_d,
                      void* stream) {
    if (!ctx || !out_d || W <= 0 || H <= 0) return MN_ERR_INVALID;
    const int64_t n = (int64_t)W * H;
    ray_directions_kernel<<<(unsigned)mn_cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(W, H, fx, fy, cx, cy, center_pixels, out_d);
    MN_LAUNCH_CHECK(ctx);
    return MN_OK;
}

int mn_rays_pairs(mn_ctx* ctx, const float* dirs_d, int64_t P, const float* c2w_d, int n_poses, const int32_t* img_idx_d,
                  const int32_t* pix_idx_d, int64_t M, float near, float far, int has_altitude, float alt_max, float alt_min,
                  float* out_d, void* stream) {
    if (!ctx || !dirs_d || !c2w_d || !img_idx_d || !pix_idx_d || !out_d || M < 0 || P < 0 || n_poses < 0) return MN_ERR_INVALID;
    if (M == 0) return MN_OK;
    rays_pairs_kernel<<<(unsigned)mn_cdiv(M, 256), 256, 0, (cudaStream_t)stream>>>(dirs_d, P, c2w_d, n_poses, img_idx_d, pix_idx_d, M, near,
                                                                                   far, has_altitude, alt_max, alt_min, out_d, ctx->status_d);
    MN_LAUNCH_CHECK(ctx);
    return MN_OK;
}

int mn_gather_batch(mn_ctx* ctx, const int64_t* idx_d, int64_t B, int64_t n_rows, const void* src0_d, int w0, void* dst0_d,
                    const void* src1_d, int w1, void* dst1_d, const void* src2_d, int w2, void* dst2_d, void* stream) {
    if (!ctx || !idx_d || B < 0 || n_rows < 0) return MN_ERR_INVALID;
    GatherArgs a{};
    const void* src[3] = {src0_d, src1_d, src2_d};
    void* dst[3] = {dst0_d, dst1_d, dst2_d};
    const int w[3] = {w0, w1, w2};
    for (int c = 0; c < 3; ++c) {
        if (!src[c]) continue;
        if (!dst[c] || w[c] < 1) return mn_fail(ctx, MN_ERR_INVALID, "mn_gather_batch: a column needs a destination and a width >= 1");
        a.src[c] = static_cast<const unsigned int*>(src[c]);
        a.dst[c] = static_cast<unsigned int*>(dst[c]);
        a.w[c] = w[c];
        a.vec[c] = w[c] % 4 == 0 && ((uintptr_t)src[c] | (uintptr_t)dst[c]) % 16 == 0;
        a.units[c] = a.vec[c] ? w[c] / 4 : w[c];
        a.row_units += a.units[c];
    }
    if (B == 0 || a.row_units == 0) return MN_OK;
    gather_batch_kernel<<<(unsigned)mn_cdiv(B * a.row_units, 256), 256, 0, (cudaStream_t)stream>>>(idx_d, B, n_rows, a, ctx->status_d);
    MN_LAUNCH_CHECK(ctx);
    return MN_OK;
}

int mn_rays(mn_ctx* ctx, const float* dirs_d, int dirs_batched, const float* c2w_d, int n_poses, int64_t P, float near,
            float far, int has_altitude, float alt_max, float alt_min, float* out_d, void* stream) {
    if (!ctx || !dirs_d || !c2w_d || !out_d) return MN_ERR_INVALID;
    const int64_t n = (int64_t)n_poses * P;
    if (n == 0) return MN_OK;
    rays_kernel<<<(unsigned)mn_cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(dirs_d, dirs_batched, c2w_d, n_poses, P, near, far,
                                                                             has_altitude, alt_max, alt_min, out_d);
    MN_LAUNCH_CHECK(ctx);
    return MN_OK;
}

int mn_sample_coarse(mn_ctx* ctx, const float* rays_d, const float* far_d, const float* z_steps_d, const float* rand_d,
                     float perturb, int64_t N, int S, float* z_out_d, float* xyz_out_d, void* stream) {
    if (!ctx || !rays_d || !z_steps_d || !z_out_d || S < 1) return MN_ERR_INVALID;
    if (perturb > 0 && !rand_d) return mn_fail(ctx, MN_ERR_INVALID, "mn_sample_coarse: perturb > 0 needs rand_d");
    if (N == 0) return MN_OK;
    sample_coarse_kernel<<<(unsigned)mn_cdiv(N * S, 256), 256, 0, (cudaStream_t)stream>>>(rays_d, far_d, z_steps_d, rand_d, perturb,
                                                                                          N, S, z_out_d, xyz_out_d);
    MN_LAUNCH_CHECK(ctx);
    return MN_OK;
}

int mn_stratify(mn_ctx* ctx, const float* z_d, int64_t z_row_stride, const float* rand_d, float perturb, int64_t N, int S,
                float* z_out_d, void* stream) {
    if (!ctx || !z_d || !z_out_d || S < 1) return MN_ERR_INVALID;
    if (perturb > 0 && !rand_d) return mn_fail(ctx, MN_ERR_INVALID, "mn_stratify: perturb > 0 needs rand_d");
    if (N == 0) return MN_OK;
    return mn_stage_stratify(ctx, z_d, z_row_stride, rand_d, perturb, N, S, 0, LiveRows{}, z_out_d, (cudaStream_t)stream);
}

int mn_points_from_z(mn_ctx* ctx, const float* rays_d, const float* z_d, int64_t N, int S, float* xyz_out_d, void* stream) {
    if (!ctx || !rays_d || !z_d || !xyz_out_d) return MN_ERR_INVALID;
    if (N == 0) return MN_OK;
    points_from_z_kernel<<<(unsigned)mn_cdiv(N * S, 256), 256, 0, (cudaStream_t)stream>>>(rays_d, z_d, N, S, xyz_out_d);
    MN_LAUNCH_CHECK(ctx);
    return MN_OK;
}

int mn_sample_pdf(mn_ctx* ctx, const float* z_coarse_d, const float* weights_d, int64_t w_stride, const float* cdf_d,
                  const float* u_d, int64_t u_row_stride, int64_t N, int S, int F, float* z_out_d, int64_t* inds_out_d,
                  float* cdf_out_d, void* stream) {
    if (!ctx || !z_coarse_d || !u_d || !z_out_d || S < 3 || F < 1) return MN_ERR_INVALID;
    if ((weights_d == nullptr) == (cdf_d == nullptr))
        return mn_fail(ctx, MN_ERR_INVALID, "mn_sample_pdf: exactly one of weights_d / cdf_d");
    if (N == 0) return MN_OK;
    return mn_stage_sample_pdf(ctx, z_coarse_d, weights_d, w_stride, cdf_d, u_d, u_row_stride, N, S, F, LiveRows{}, z_out_d, inds_out_d,
                               cdf_out_d, (cudaStream_t)stream);
}

int mn_sort_cat(mn_ctx* ctx, const float* a_d, int na, const float* b_d, int nb, int64_t N, int descending, float* out_d,
                void* stream) {
    if (!ctx || !a_d || (nb > 0 && !b_d) || !out_d) return MN_ERR_INVALID;
    if (N == 0) return MN_OK;
    return mn_stage_sort_cat(ctx, a_d, na, b_d, nb, N, descending, LiveRows{}, out_d, nullptr, (cudaStream_t)stream);
}

int mn_composite(mn_ctx* ctx, const float* raw_d, const float* z_d, const float* depth_real_d, int S, const float* raw2_d,
                 const float* z2_d, const float* depth_real2_d, int S2, const float* last_delta_d, int64_t N, int flip,
                 float* weights_out_d, float* rgb_out_d, float* depth_out_d, float* depth_var_out_d, float* bg_lambda_out_d,
                 void* stream) {
    if (!ctx || !raw_d || !z_d || !last_delta_d || S < 1 || S2 < 0) return MN_ERR_INVALID;
    if (S2 > 0 && (!raw2_d || !z2_d)) return MN_ERR_INVALID;
    if (depth_real_d && S2 > 0 && !depth_real2_d) return MN_ERR_INVALID;
    if (N == 0) return MN_OK;
    return mn_stage_composite(ctx, raw_d, z_d, depth_real_d, S, raw2_d, z2_d, depth_real2_d, S2, last_delta_d, N, flip, LiveRows{},
                              weights_out_d, rgb_out_d, depth_out_d, depth_var_out_d, bg_lambda_out_d, (cudaStream_t)stream);
}

int mn_composite_backward(mn_ctx* ctx, const float* raw_d, const float* z_d, int S, const float* raw2_d, const float* z2_d,
                          int S2, const float* last_delta_d, int64_t N, int flip, const float* grad_rgb_d,
                          const float* grad_lambda_d, float* grad_raw_d, float* grad_raw2_d, void* stream) {
    if (!ctx || !raw_d || !z_d || !last_delta_d || !grad_rgb_d || !grad_raw_d || S < 1 || S2 < 0) return MN_ERR_INVALID;
    if (S2 > 0 && (!raw2_d || !z2_d || !grad_raw2_d)) return MN_ERR_INVALID;
    if (N == 0) return MN_OK;
    return mn_stage_composite_backward(ctx, raw_d, z_d, S, raw2_d, z2_d, S2, last_delta_d, N, flip, LiveRows{}, grad_rgb_d, grad_lambda_d,
                                       grad_raw_d, grad_raw2_d, (cudaStream_t)stream);
}

int mn_sh_to_rgb_backward(mn_ctx* ctx, int deg, const float* coef_d, int64_t coef_stride, const float* dirs_d,
                          int64_t dir_stride, int dir_div, int64_t B, int apply_sigmoid, const float* grad_out_d,
                          float* grad_coef_d, void* stream) {
    if (!ctx || !coef_d || !dirs_d || !grad_out_d || !grad_coef_d || deg < 0 || deg > 4 || dir_div < 1) return MN_ERR_INVALID;
    if (B == 0) return MN_OK;
    return mn_stage_sh_to_rgb_backward(ctx, deg, coef_d, coef_stride, dirs_d, dir_stride, dir_div, B, apply_sigmoid, LiveRows{}, grad_out_d,
                                       grad_coef_d, (cudaStream_t)stream);
}

int mn_intersect_sphere(mn_ctx* ctx, const float* rays_d, const float* center3_d, const float* radius3_d, int64_t N,
                        float* fg_far_out_d, void* stream) {
    if (!ctx || !rays_d || !fg_far_out_d) return MN_ERR_INVALID;
    if (radius3_d && !center3_d) return MN_ERR_INVALID;
    if (N == 0) return MN_OK;
    intersect_sphere_kernel<<<(unsigned)mn_cdiv(N, 256), 256, 0, (cudaStream_t)stream>>>(rays_d, center3_d, radius3_d, N,
                                                                                         fg_far_out_d, ctx->status_d);
    MN_LAUNCH_CHECK(ctx);
    return MN_OK;
}

int mn_points_outside(mn_ctx* ctx, const float* rays_d, const int64_t* ray_ids_d, const float* depth_d, const float* center3_d,
                      const float* radius3_d, int64_t n, int S, int include_xyz_real, int cluster_2d, float* pts_out_d,
                      float* depth_real_out_d, void* stream) {
    if (!ctx || !rays_d || !depth_d || !pts_out_d || !depth_real_out_d) return MN_ERR_INVALID;
    if (n == 0) return MN_OK;
    return mn_stage_points_outside(ctx, rays_d, ray_ids_d, depth_d, center3_d, radius3_d, n, S, include_xyz_real, cluster_2d, 0,
                                   LiveRows{}, pts_out_d, depth_real_out_d, (cudaStream_t)stream);
}

int mn_sh_to_rgb(mn_ctx* ctx, int deg, const float* coef_d, int64_t coef_stride, const float* dirs_d, int64_t dir_stride,
                 int dir_div, int64_t B, int apply_sigmoid, float* out_d, void* stream) {
    if (!ctx || !coef_d || !dirs_d || !out_d || deg < 0 || deg > 4 || dir_div < 1) return MN_ERR_INVALID;
    if (B == 0) return MN_OK;
    return mn_stage_sh_to_rgb(ctx, deg, coef_d, coef_stride, dirs_d, dir_stride, dir_div, B, apply_sigmoid, LiveRows{}, out_d,
                              (cudaStream_t)stream);
}

int mn_embed(mn_ctx* ctx, const float* x_d, int64_t B, int dim, int n_freqs, float* out_d, void* stream) {
    if (!ctx || !x_d || !out_d || dim < 1 || n_freqs < 0) return MN_ERR_INVALID;
    if (B == 0) return MN_OK;
    const int64_t n = B * dim * (1 + n_freqs);
    embed_kernel<<<(unsigned)mn_cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(x_d, B, dim, n_freqs, out_d);
    MN_LAUNCH_CHECK(ctx);
    return MN_OK;
}

}  // extern "C"

// ---- the one launch of each stage kernel (mn_model.cuh): the public entry points above validate and call these; the render
// passes of mn_render_rays(_bg) call them directly, the background pass with its device ray count and sample-order options ----
int mn_stage_stratify(mn_ctx* ctx, const float* z_d, int64_t z_row_stride, const float* rand_d, float perturb, int64_t N, int S, int flip,
                      LiveRows live, float* z_out_d, cudaStream_t st) {
    stratify_kernel<<<(unsigned)mn_cdiv(N * S, 256), 256, 0, st>>>(z_d, z_row_stride, rand_d, perturb, N, S, z_out_d, live, flip);
    MN_LAUNCH_CHECK(ctx);
    return MN_OK;
}

int mn_stage_points_outside(mn_ctx* ctx, const float* rays_d, const int64_t* ray_ids_d, const float* depth_d, const float* center3_d,
                            const float* radius3_d, int64_t n, int S, int include_xyz_real, int cluster_2d, int flip_pts, LiveRows live,
                            float* pts_out_d, float* depth_real_out_d, cudaStream_t st) {
    points_outside_kernel<<<(unsigned)mn_cdiv(n * S, 256), 256, 0, st>>>(rays_d, ray_ids_d, depth_d, center3_d, radius3_d, n, S,
                                                                         include_xyz_real, cluster_2d, pts_out_d, depth_real_out_d,
                                                                         live, flip_pts);
    MN_LAUNCH_CHECK(ctx);
    return MN_OK;
}

int mn_stage_sample_pdf(mn_ctx* ctx, const float* z_coarse_d, const float* weights_d, int64_t w_stride, const float* cdf_d, const float* u_d,
                        int64_t u_row_stride, int64_t N, int S, int F, LiveRows live, float* z_out_d, int64_t* inds_out_d,
                        float* cdf_out_d, cudaStream_t st) {
    if (S < 3 || F < 1) return mn_fail(ctx, MN_ERR_INVALID, "mn_sample_pdf: resampling needs >= 3 coarse samples and >= 1 draw");
    const size_t sm = (size_t)4 * 2 * S * sizeof(float);
    if (sm > 200 * 1024) return mn_fail(ctx, MN_ERR_UNSUPPORTED, "mn_sample_pdf: too many coarse samples");
    MN_CUDA(ctx, cudaFuncSetAttribute(sample_pdf_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
    sample_pdf_kernel<<<(unsigned)mn_cdiv(N, 4), 128, sm, st>>>(z_coarse_d, weights_d, w_stride, cdf_d, u_d, u_row_stride, N, S, F, z_out_d,
                                                                 inds_out_d, cdf_out_d, live);
    MN_LAUNCH_CHECK(ctx);
    return MN_OK;
}

int mn_stage_sort_cat(mn_ctx* ctx, const float* a_d, int na, const float* b_d, int nb, int64_t N, int descending, LiveRows live,
                      float* out_d, float* out_flip_d, cudaStream_t st) {
    const int npad = pow2_at_least(na + nb);
    if (npad > 4096) return mn_fail(ctx, MN_ERR_UNSUPPORTED, "mn_sort_cat: more than 4096 samples per ray");
    const size_t sm = (size_t)4 * npad * (sizeof(float) + sizeof(unsigned short));
    MN_CUDA(ctx, cudaFuncSetAttribute(sort_cat_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
    sort_cat_kernel<<<(unsigned)mn_cdiv(N, 4), 128, sm, st>>>(a_d, na, b_d, nb, N, descending, npad, out_d, out_flip_d, live);
    MN_LAUNCH_CHECK(ctx);
    return MN_OK;
}

int mn_stage_composite(mn_ctx* ctx, const float* raw_d, const float* z_d, const float* depth_real_d, int S, const float* raw2_d,
                       const float* z2_d, const float* depth_real2_d, int S2, const float* last_delta_d, int64_t N, int flip,
                       LiveRows live, float* weights_out_d, float* rgb_out_d, float* depth_out_d, float* depth_var_out_d,
                       float* bg_lambda_out_d, cudaStream_t st) {
    CompositeArgs a{};
    a.raw = raw_d; a.z = z_d; a.dreal = depth_real_d; a.S = S;
    a.raw2 = raw2_d; a.z2 = z2_d; a.dreal2 = depth_real2_d; a.S2 = S2;
    a.last_delta = last_delta_d; a.N = N; a.flip = flip;
    a.weights = weights_out_d; a.rgb = rgb_out_d; a.depth = depth_out_d; a.var = depth_var_out_d; a.lambda = bg_lambda_out_d;
    a.live = live;
    return composite_launch(ctx, composite_kernel, a, "mn_composite", st);
}

int mn_stage_sh_to_rgb(mn_ctx* ctx, int deg, const float* coef_d, int64_t coef_stride, const float* dirs_d, int64_t dir_stride,
                       int dir_div, int64_t B, int apply_sigmoid, LiveRows live, float* out_d, cudaStream_t st, const int* gather) {
    sh_to_rgb_kernel<<<(unsigned)mn_cdiv(B, 256), 256, 0, st>>>(deg, coef_d, coef_stride, dirs_d, dir_stride, dir_div, B, apply_sigmoid,
                                                                out_d, live, gather);
    MN_LAUNCH_CHECK(ctx);
    return MN_OK;
}

int mn_stage_composite_backward(mn_ctx* ctx, const float* raw_d, const float* z_d, int S, const float* raw2_d, const float* z2_d, int S2,
                                const float* last_delta_d, int64_t N, int flip, LiveRows live, const float* grad_rgb_d,
                                const float* grad_lambda_d, float* grad_raw_d, float* grad_raw2_d, cudaStream_t st) {
    CompositeBwdArgs a{};
    a.raw = raw_d; a.z = z_d; a.S = S;
    a.raw2 = raw2_d; a.z2 = z2_d; a.S2 = S2;
    a.last_delta = last_delta_d; a.N = N; a.flip = flip;
    a.grad_rgb = grad_rgb_d; a.grad_lambda = grad_lambda_d;
    a.grad_raw = grad_raw_d; a.grad_raw2 = grad_raw2_d;
    a.live = live;
    return composite_launch(ctx, composite_bwd_kernel, a, "mn_composite_backward", st);
}

int mn_stage_sh_to_rgb_backward(mn_ctx* ctx, int deg, const float* coef_d, int64_t coef_stride, const float* dirs_d, int64_t dir_stride,
                                int dir_div, int64_t B, int apply_sigmoid, LiveRows live, const float* grad_out_d, float* grad_coef_d,
                                cudaStream_t st, const int* gather) {
    sh_to_rgb_bwd_kernel<<<(unsigned)mn_cdiv(B, 256), 256, 0, st>>>(deg, coef_d, coef_stride, dirs_d, dir_stride, dir_div, B, apply_sigmoid,
                                                                    grad_out_d, grad_coef_d, live, gather);
    MN_LAUNCH_CHECK(ctx);
    return MN_OK;
}
