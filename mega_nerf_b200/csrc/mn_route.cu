// Spatial routing of sample rows to sub-modules (models/mega_nerf.py:21-49), bucketed into
// MN_TILE-aligned slot ranges so that every MLP tile belongs to exactly one sub-module, plus the
// ascending-sub-module blend that replaces `results[mask] += sub_result * weights`.
//
// Distances restate torch.cdist's matmul path bit for bit (SURVEY.md §8c / §9-Q3):
//   x_ = [-2x, |x|^2, 1],  c_ = [c, 1, |c|^2],  d^2 = FMA chain over k ascending from an accumulator
//   of 0, clamp_min(0), sqrt.  Batches with <= 25 rows AND <= 25 centroids take cdist's direct path
//   sqrt(fma-accumulated sum (x-c)^2) instead, as torch does.
#include "mn_model.cuh"

namespace {

// `prune` > 0 (the routing kernels; = max(boundary_margin, 1)^2): centroids whose SQUARED distance exceeds prune x (1 + 1e-5) x the
// smallest squared distance can neither be the nearest nor fall inside the margin - sqrt is monotone and the slack covers its
// rounding 50 times over - so their distance is reported as +inf without the IEEE sqrt (and, downstream, without the two IEEE
// divisions of the blend weight).  Every value that takes part in a comparison or a weight is computed exactly as before.
template <int KMAX>
__device__ __forceinline__ void distances(const RowSrc& src, int64_t row, const float* __restrict__ cent, int K,
                                          int s, bool direct, float* d, float prune = 0.0f) {
    float x[3];
    for (int j = s; j < 3; ++j) x[j] = src.route_xyz(row, j);
    if (direct) {
#pragma unroll
        for (int k = 0; k < KMAX; ++k) {
            if (k >= K) break;
            float acc = 0.0f;
            for (int j = s; j < 3; ++j) {
                const float t = x[j] - cent[k * 3 + j];
                acc = fmaf(t, t, acc);  // torch's direct cdist kernel contracts this (probe: 100% bitwise)
            }
            d[k] = sqrtf(acc);
        }
        return;
    }
    float xn = x[s] * x[s];
    for (int j = s + 1; j < 3; ++j) xn = xn + x[j] * x[j];
    float amin = INFINITY;
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
        if (k >= K) break;
        float cn = cent[k * 3 + s] * cent[k * 3 + s];
        for (int j = s + 1; j < 3; ++j) cn = cn + cent[k * 3 + j] * cent[k * 3 + j];
        float acc = 0.0f;
        for (int j = s; j < 3; ++j) acc = fmaf(-2.0f * x[j], cent[k * 3 + j], acc);
        acc = fmaf(xn, 1.0f, acc);
        acc = fmaf(1.0f, cn, acc);
        acc = fmaxf(acc, 0.0f);
        d[k] = acc;
        amin = fminf(amin, acc);
    }
    const float bound = prune > 0.0f ? fmaf(prune * 1.00001f, amin, 1e-30f) : INFINITY;
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
        if (k >= K) break;
        d[k] = d[k] > bound ? INFINITY : sqrtf(d[k]);
    }
}

// -> number of active sub-modules; mask bits; for margin > 1 the normalised weights in w[]
template <int KMAX>
__device__ __forceinline__ uint64_t route_row(const float* d, int K, float margin, float* w) {
    float dmin = d[0];
    int amin = 0;
#pragma unroll
    for (int k = 1; k < KMAX; ++k)
        if (k < K && d[k] < dmin) { dmin = d[k]; amin = k; }
    if (!(margin > 1.0f)) return 1ull << amin;
    uint64_t mask = 0;
    float sum = 0.0f;
    const float thr = margin * dmin;
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
        if (k < K) {
            float inv = 0.0f;
            if (!(d[k] > thr)) inv = 1.0f / (d[k] + 1e-8f);       // the reference masks 1/(d + 1e-8) with d > thr: same values, fewer divisions
            w[k] = inv;
            sum = sum + inv;
        }
    }
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
        if (k < K) {
            if (w[k] != 0.0f) w[k] = w[k] / sum;                   // 0 / sum == 0
            if (w[k] > 0.0f) mask |= 1ull << k;
        }
    }
    return mask;
}

// The routing decision (distances, threshold, normalised weights: ~2000 instructions per row with IEEE sqrt / div) is
// made ONCE, here; the scatter pass re-reads the active-set mask [B] and the blend weights [K][B] (active entries only).
// Rows at or past live.rows(B) (a call whose row count lives on the device) are not routed; cdist's direct path follows that
// count, as it follows the batch size in the reference.
template <int KMAX>
__global__ void route_count_kernel(RowSrc src, int64_t B, LiveRows live, const float* __restrict__ cent, int K, int s, float margin,
                                   int64_t cap, int* counters, unsigned long long* __restrict__ mask_out, float* __restrict__ w_out) {
    __shared__ int hist[MN_MAX_SUB];
    __shared__ float sc[MN_MAX_SUB * 3];
    for (int i = threadIdx.x; i < K * 3; i += blockDim.x) sc[i] = cent[i];
    for (int i = threadIdx.x; i < K; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    const int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t n = live.rows(B);
    const bool direct = n <= 25 && K <= 25;
    uint64_t mask = 0;
    if (row < n) {
        float d[KMAX], w[KMAX];
        distances<KMAX>(src, row, sc, K, s, direct, d, margin > 1.0f ? margin * margin : 1.0f);
        mask = route_row<KMAX>(d, K, margin, w);
        mask_out[row] = mask;
        if (w_out) {
#pragma unroll
            for (int k = 0; k < KMAX; ++k)
                if (k < K && ((mask >> k) & 1)) w_out[(int64_t)k * B + row] = w[k];
        }
    }
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
        if (k >= K) break;
        const unsigned b = __ballot_sync(0xffffffffu, (mask >> k) & 1);
        if ((threadIdx.x & 31) == 0 && b) atomicAdd(&hist[k], __popc(b));
    }
    __syncthreads();
    for (int i = threadIdx.x; i < K; i += blockDim.x)
        if (hist[i]) atomicAdd(&counters[CNT_COUNT + i], hist[i]);
    // the last block to finish turns the counts into bucket offsets (was a separate 1-thread launch)
    __shared__ int last;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) last = atomicAdd(&counters[CNT_TICKET], 1) == (int)gridDim.x - 1;
    __syncthreads();
    if (last && threadIdx.x == 0) {
        __threadfence();
        int off = 0, pairs = 0;
        for (int k = 0; k < K; ++k) {
            counters[CNT_START + k] = off;
            const int c = *(volatile int*)&counters[CNT_COUNT + k];
            pairs += c;
            off += (c + MN_BUCKET - 1) / MN_BUCKET * MN_BUCKET;
            counters[CNT_CURSOR + k] = 0;
        }
        counters[CNT_START + K] = off;
        // the MLP kernels walk the tiles below CNT_NSLOTS: past the slot capacity (an overflow, whose pairs the scatter pass drops)
        // there is no slot, image or output to read or write
        counters[CNT_NSLOTS] = off < cap ? off : (int)cap;
        counters[CNT_NPAIRS] = pairs;
    }
}

template <int KMAX>
__global__ void route_scatter_kernel(int64_t B, LiveRows live, int K, int* counters, int64_t cap,
                                     const unsigned long long* __restrict__ mask_in, const float* __restrict__ w_in, int* slot_row,
                                     float* slot_w, int* row_slots, unsigned int* status) {
    const int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    const int64_t n = live.rows(B);
    const uint64_t mask = row < n ? mask_in[row] : 0ull;
    // one global atomic per (block, sub-module): warp ballots -> shared per-warp counts -> block prefix
    __shared__ int wcnt[8][KMAX];     // blockDim.x == 256
    const int warp = threadIdx.x >> 5;
    unsigned bal[KMAX];
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
        bal[k] = 0;
        if (k < K) {
            bal[k] = __ballot_sync(0xffffffffu, (mask >> k) & 1);
            if (lane == 0) wcnt[warp][k] = __popc(bal[k]);
        }
    }
    __syncthreads();
    if (threadIdx.x < K) {
        const int k = threadIdx.x;
        int tot = 0;
        for (int wi = 0; wi < 8; ++wi) tot += wcnt[wi][k];
        int base = tot ? atomicAdd(&counters[CNT_CURSOR + k], tot) : 0;
        base += counters[CNT_START + k];
        for (int wi = 0; wi < 8; ++wi) {
            const int c = wcnt[wi][k];
            wcnt[wi][k] = base;
            base += c;
        }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
        if (k >= K) break;
        int slot = -1;
        if ((mask >> k) & 1) {
            slot = wcnt[warp][k] + __popc(bal[k] & ((1u << lane) - 1));
            if (slot >= cap) {
                // slot capacity exceeded (more (row, sub-module) pairs than B x max_multiplicity): the contribution cannot be
                // computed.  Loud in the data - combine_kernel turns the row into NaN, which the reference's Runner rejects
                // (runner.py:260-261) - and in the sticky status word (MN_ERR_WORKSPACE at the next mn_check_status).
                atomicOr(status, MN_STATUS_OVERFLOW);
                slot = -2;
            } else {
                slot_row[slot] = (int)row;
                if (slot_w) slot_w[slot] = w_in[(int64_t)k * B + row];
            }
        }
        if (row < n && row_slots) row_slots[row * K + k] = slot;
    }
}

__global__ void combine_kernel(int64_t B, LiveRows live, int K, const int* __restrict__ row_slots, const float* __restrict__ slot_out,
                               int out_cols, float* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= live.rows(B) * out_cols) return;
    const int64_t row = i / out_cols;
    const int c = (int)(i % out_cols);
    float acc = 0.0f;
    for (int k = 0; k < K; ++k) {  // ascending sub-module order (mega_nerf.py:34,49)
        const int slot = row_slots[row * K + k];
        if (slot >= 0) acc = acc + slot_out[(int64_t)slot * out_cols + c];
        else if (slot == -2) acc = __int_as_float(0x7fc00000);   // dropped contribution (capacity overflow): poison, never a silent wrong blend
    }
    out[i] = acc;
}

template <int KMAX>
__global__ void route_only_kernel(RowSrc src, int64_t B, const float* __restrict__ cent, int K, int s, float margin,
                                  int direct, int* assign, float* weights) {
    const int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= B) return;
    float d[KMAX], w[KMAX];
    distances<KMAX>(src, row, cent, K, s, direct, d, margin > 1.0f ? margin * margin : 1.0f);
    const uint64_t mask = route_row<KMAX>(d, K, margin, w);
    if (margin > 1.0f) {
#pragma unroll
        for (int k = 0; k < KMAX; ++k)
            if (k < K) weights[row * K + k] = w[k];
    } else {
        assign[row] = __ffsll((long long)mask) - 1;
    }
}


// ------------------------------------------------------------------------------------------------
// Cluster masks (scripts/create_cluster_masks.py:155-201; SURVEY.md §8f-3): for every ray the minimum over
// its S samples of d(sample, centroid_k) / (min_j d(sample, centroid_j) + 1e-8), without materialising
// the reference's [rays, S, K] distance tensor.  One warp per ray, lanes stride the samples, running
// minima in registers, one shuffle reduction at the end.  Arithmetic = the torch ops, separately rounded:
// z = near (1 - t) + far t;  xyz = o + d z;  cdist's matmul path (FMA chain, see distances<> above).
// ------------------------------------------------------------------------------------------------
template <int KMAX>
__global__ void __launch_bounds__(128) cluster_ratio_kernel(const float* __restrict__ rays, int64_t N,
                                                            const float* __restrict__ z_steps, int S,
                                                            const float* __restrict__ cent, int K, int s, float margin,
                                                            float* __restrict__ ratios, unsigned char* __restrict__ mask) {
    __shared__ float sc[MN_MAX_SUB * 3];
    __shared__ float scn[MN_MAX_SUB];
    for (int i = threadIdx.x; i < K * 3; i += blockDim.x) sc[i] = cent[i];
    __syncthreads();
    for (int k = threadIdx.x; k < K; k += blockDim.x) {
        float cn = sc[k * 3 + s] * sc[k * 3 + s];
        for (int j = s + 1; j < 3; ++j) cn = cn + sc[k * 3 + j] * sc[k * 3 + j];
        scn[k] = cn;
    }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t ray = (int64_t)blockIdx.x * 4 + warp;
    if (ray >= N) return;
    const float* r = rays + ray * 8;
    const float o[3] = {r[0], r[1], r[2]}, dir[3] = {r[3], r[4], r[5]};
    const float near = r[6], far = r[7];
    float best[KMAX];
#pragma unroll
    for (int k = 0; k < KMAX; ++k) best[k] = INFINITY;
    for (int i = lane; i < S; i += 32) {
        const float t = z_steps[i];
        const float z = near * (1.0f - t) + far * t;
        float x[3];
        for (int j = 0; j < 3; ++j) x[j] = o[j] + dir[j] * z;
        float xn = x[s] * x[s];
        for (int j = s + 1; j < 3; ++j) xn = xn + x[j] * x[j];
        float d[KMAX];
        float dmin = INFINITY;
#pragma unroll
        for (int k = 0; k < KMAX; ++k) {
            if (k < K) {
                float acc = 0.0f;
                for (int j = s; j < 3; ++j) acc = fmaf(-2.0f * x[j], sc[k * 3 + j], acc);
                acc = fmaf(xn, 1.0f, acc);
                acc = fmaf(1.0f, scn[k], acc);
                d[k] = sqrtf(fmaxf(acc, 0.0f));
                dmin = fminf(dmin, d[k]);
            }
        }
        const float den = dmin + 1e-8f;
#pragma unroll
        for (int k = 0; k < KMAX; ++k)
            if (k < K) best[k] = fminf(best[k], d[k] / den);
    }
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
        if (k < K) {
            float v = best[k];
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, off));
            if (lane == 0) {
                if (ratios) ratios[ray * K + k] = v;
                if (mask) mask[(int64_t)k * N + ray] = v <= margin ? 1 : 0;
            }
        }
    }
}

}  // namespace

size_t mn_route_scratch_bytes(const mn_model* m, int64_t B) {
    size_t n = mn_align((size_t)B * sizeof(unsigned long long));                                   // active-set masks
    if (m->d.boundary_margin > 1.0f) n += mn_align((size_t)B * (size_t)m->d.n_sub * sizeof(float));   // blend weights [K][B]
    return n;
}

int mn_route_build(mn_ctx* ctx, mn_model* m, const RowSrc& src, int64_t B, LiveRows live, int64_t cap, int* slot_row, float* slot_w,
                   int* row_slots, void* scratch, cudaStream_t st) {
    unsigned long long* mask_buf = reinterpret_cast<unsigned long long*>(scratch);
    float* w_buf = m->d.boundary_margin > 1.0f
                       ? reinterpret_cast<float*>(reinterpret_cast<char*>(scratch) + mn_align((size_t)B * sizeof(unsigned long long)))
                       : nullptr;
    const int K = m->d.n_sub;
    MN_CUDA(ctx, cudaMemsetAsync(m->counters_d, 0, CNT_TOTAL * sizeof(int), st));
    MN_CUDA(ctx, cudaMemsetAsync(slot_row, 0xFF, (size_t)cap * sizeof(int), st));
    const unsigned blocks = (unsigned)mn_cdiv(B, 256);
#define MN_ROUTE_DISPATCH(KERNEL, GRID, BLOCK, ...)                                   \
    do {                                                                              \
        if (K <= 8) KERNEL<8><<<GRID, BLOCK, 0, st>>>(__VA_ARGS__);                   \
        else if (K <= 32) KERNEL<32><<<GRID, BLOCK, 0, st>>>(__VA_ARGS__);            \
        else KERNEL<MN_MAX_SUB><<<GRID, BLOCK, 0, st>>>(__VA_ARGS__);                 \
    } while (0)
    MN_ROUTE_DISPATCH(route_count_kernel, blocks, 256, src, B, live, m->centroids_d, K, m->d.cluster_dim_start, m->d.boundary_margin,
                      cap, m->counters_d, mask_buf, w_buf);
    MN_LAUNCH_CHECK(ctx);
    MN_ROUTE_DISPATCH(route_scatter_kernel, blocks, 256, B, live, K, m->counters_d, cap, mask_buf, w_buf, slot_row, slot_w, row_slots,
                      ctx->status_d);
    MN_LAUNCH_CHECK(ctx);
    return MN_OK;
}

int mn_route_combine(mn_ctx* ctx, mn_model* m, int64_t B, LiveRows live, const int* row_slots, const float* slot_out, int out_cols,
                     float* out, cudaStream_t st) {
    const int64_t n = B * out_cols;
    combine_kernel<<<(unsigned)mn_cdiv(n, 256), 256, 0, st>>>(B, live, m->d.n_sub, row_slots, slot_out, out_cols, out);
    MN_LAUNCH_CHECK(ctx);
    return MN_OK;
}

extern "C" int mn_model_route(mn_ctx* ctx, mn_model* m, const mn_rows* rows, int64_t B, int32_t* assign_out_d,
                              float* weights_out_d, void* stream) {
    if (!ctx || !m || !rows) return MN_ERR_INVALID;
    if (m->d.kind != 2) return mn_fail(ctx, MN_ERR_INVALID, "mn_model_route: not a MegaNeRF model");
    RowSrc src{};
    src.x = rows->x_d;
    src.cols = rows->cols;
    src.div = 1;
    const int K = m->d.n_sub;
    const int direct = (B <= 25 && K <= 25) ? 1 : 0;
    if (B == 0) return MN_OK;
    cudaStream_t st = (cudaStream_t)stream;
    MN_ROUTE_DISPATCH(route_only_kernel, (unsigned)mn_cdiv(B, 128), 128, src, B, m->centroids_d, K, m->d.cluster_dim_start,
                      m->d.boundary_margin, direct, assign_out_d, weights_out_d);
    MN_LAUNCH_CHECK(ctx);
    return MN_OK;
}

extern "C" int mn_cluster_min_dist_ratios(mn_ctx* ctx, const float* rays_d, int64_t N, const float* z_steps_d, int S,
                                          const float* centroids_d, int K, int cluster_2d, float boundary_margin,
                                          float* ratios_out_d, unsigned char* mask_out_d, void* stream) {
    if (!ctx || !rays_d || !z_steps_d || !centroids_d || N < 0 || S < 1 || K < 1 || K > MN_MAX_SUB) return MN_ERR_INVALID;
    if (!ratios_out_d && !mask_out_d) return MN_ERR_INVALID;
    if (N == 0) return MN_OK;
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned blocks = (unsigned)mn_cdiv(N, 4);
    const int s = cluster_2d ? 1 : 0;
    MN_ROUTE_DISPATCH(cluster_ratio_kernel, blocks, 128, rays_d, N, z_steps_d, S, centroids_d, K, s, boundary_margin,
                      ratios_out_d, mask_out_d);
    MN_LAUNCH_CHECK(ctx);
    return MN_OK;
}
