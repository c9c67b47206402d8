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

// Adds this block's rows (`mask`: one bit per sub-module) to the per-sub-module counts; the last block to finish turns the
// counts into MN_BUCKET-aligned bucket offsets.  `hist` is the block's zeroed shared histogram [K]; every thread calls this.
template <int KMAX>
__device__ __forceinline__ void bucket_count(uint64_t mask, int K, int64_t cap, int* counters, int* hist) {
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
    // the queried samples of an occupancy grid (src.gather) stand for the whole B-row query, whose batch size picks the path
    const bool direct = (src.gather ? B : n) <= 25 && K <= 25;
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
    bucket_count<KMAX>(mask, K, cap, counters, hist);
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

// ------------------------------------------------------------------------------------------------
// Expert-parallel query (mega_nerf_b200/expert_parallel.py): the (row, sub-module) pairs of one query in the order of
// plan_dispatch - destination rank (k mod world), sub-module, row - written straight into `world` fixed-capacity segments.
// Rows ascend inside a sub-module because every block owns EP_ROWS consecutive rows and ranks its pairs by warp and lane:
// pass 1 counts per (block, sub-module), its last block scans those counts over the blocks; pass 2 places the pairs.
// ------------------------------------------------------------------------------------------------
#define EP_ROWS 512     // rows (= threads) per block of both dispatch passes

// active sub-modules of a row from the router's output: the assignment (hard routing) or the non-zero blend weights
template <int KMAX>
__device__ __forceinline__ uint64_t ep_row_mask(const int* __restrict__ assign, const float* __restrict__ w, int64_t row, int K) {
    if (assign) return 1ull << assign[row];
    uint64_t mask = 0;
#pragma unroll
    for (int k = 0; k < KMAX; ++k)
        if (k < K && w[row * K + k] > 0.0f) mask |= 1ull << k;
    return mask;
}

// Scan state of a dispatch (workspace): blk [n_blocks][K] per-block counts, turned into the block's first position among its
// sub-module's pairs; start [K] position of a sub-module's first pair inside its segment; seg [world] pairs per segment.
struct EpScan {
    int* blk;
    int* start;
    int* seg;
    int* ticket;
};

template <int KMAX>
__global__ void __launch_bounds__(EP_ROWS) ep_count_kernel(const int* __restrict__ assign, const float* __restrict__ w, int64_t B,
                                                           int K, int world, EpScan s, int* __restrict__ counts) {
    __shared__ int wcnt[EP_ROWS / 32][KMAX];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t row = (int64_t)blockIdx.x * EP_ROWS + threadIdx.x;
    const uint64_t mask = row < B ? ep_row_mask<KMAX>(assign, w, row, K) : 0ull;
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
        if (k >= K) break;
        const unsigned b = __ballot_sync(0xffffffffu, (mask >> k) & 1);
        if (lane == 0) wcnt[warp][k] = __popc(b);
    }
    __syncthreads();
    for (int k = threadIdx.x; k < K; k += blockDim.x) {
        int tot = 0;
        for (int wi = 0; wi < EP_ROWS / 32; ++wi) tot += wcnt[wi][k];
        s.blk[(int64_t)blockIdx.x * K + k] = tot;
    }
    __shared__ int last;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) last = atomicAdd(s.ticket, 1) == (int)gridDim.x - 1;
    __syncthreads();
    if (!last) return;
    __threadfence();
    // exclusive scan of every sub-module's column over the blocks: one warp per sub-module, 32 blocks per step
    __shared__ int total[KMAX];
    volatile int* blk = s.blk;
    for (int k = warp; k < K; k += EP_ROWS / 32) {
        int carry = 0;
        for (int b0 = 0; b0 < (int)gridDim.x; b0 += 32) {
            const int b = b0 + lane;
            const int v = b < (int)gridDim.x ? blk[(int64_t)b * K + k] : 0;
            int inc = v;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int t = __shfl_up_sync(0xffffffffu, inc, o);
                if (lane >= o) inc += t;
            }
            if (b < (int)gridDim.x) blk[(int64_t)b * K + k] = carry + inc - v;
            carry += __shfl_sync(0xffffffffu, inc, 31);
        }
        if (lane == 0) total[k] = carry;
    }
    __syncthreads();
    // segment layout: the sub-modules of destination d in ascending order; counts [world][K] (0 where d does not own k)
    for (int d = threadIdx.x; d < world; d += blockDim.x) {
        int off = 0;
        for (int k = d; k < K; k += world) {
            s.start[k] = off;
            off += total[k];
        }
        s.seg[d] = off;
    }
    for (int i = threadIdx.x; i < world * K; i += blockDim.x) {
        const int d = i / K, k = i % K;
        counts[i] = k % world == d ? total[k] : 0;
    }
}

// Pass 2: pair p of segment d goes to slot d * cap + p: payload row (child input, sub-module id, density noise), home-side
// row and blend weight, and the row's slot per sub-module for the combine (-1 none, -2 past the segment: poisons the row).
// The unused tail of every segment gets id -1 (payload) and row -1.
template <int KMAX>
__global__ void __launch_bounds__(EP_ROWS) ep_scatter_kernel(const float* __restrict__ x, int64_t B, int xcols, int xoff,
                                                             const int* __restrict__ assign, const float* __restrict__ w,
                                                             const float* __restrict__ noise, int K, int world, int64_t cap,
                                                             EpScan s, float* __restrict__ send, int* __restrict__ pair_row,
                                                             float* __restrict__ pair_w, int* __restrict__ row_slots,
                                                             unsigned int* status) {
    __shared__ int wbase[EP_ROWS / 32][KMAX];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t row = (int64_t)blockIdx.x * EP_ROWS + threadIdx.x;
    const uint64_t mask = row < B ? ep_row_mask<KMAX>(assign, w, row, K) : 0ull;
    const int c_in = xcols - xoff, width = c_in + 1 + (noise ? 1 : 0);
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
        if (k >= K) break;
        const unsigned b = __ballot_sync(0xffffffffu, (mask >> k) & 1);
        if (lane == 0) wbase[warp][k] = __popc(b);
    }
    __syncthreads();
    for (int k = threadIdx.x; k < K; k += blockDim.x) {
        int base = s.start[k] + s.blk[(int64_t)blockIdx.x * K + k];
        for (int wi = 0; wi < EP_ROWS / 32; ++wi) {
            const int c = wbase[wi][k];
            wbase[wi][k] = base;
            base += c;
        }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
        if (k >= K) break;
        const unsigned b = __ballot_sync(0xffffffffu, (mask >> k) & 1);
        if (row >= B) continue;
        int64_t slot = -1;
        if ((mask >> k) & 1) {
            const int64_t p = wbase[warp][k] + __popc(b & ((1u << lane) - 1));
            if (p >= cap) {
                atomicOr(status, MN_STATUS_OVERFLOW);      // more pairs than B x max_multiplicity (mn_model_set_max_multiplicity)
                slot = -2;
            } else {
                slot = (int64_t)(k % world) * cap + p;
                float* dst = send + slot * width;
                const float* src = x + row * xcols + xoff;
                for (int j = 0; j < c_in; ++j) dst[j] = src[j];
                dst[c_in] = (float)k;
                if (noise) dst[c_in + 1] = noise[row];
                pair_row[slot] = (int)row;
                if (w) pair_w[slot] = w[row * K + k];
            }
        }
        if (w) row_slots[row * K + k] = (int)slot;
        else if (slot != -1) row_slots[row] = (int)slot;
    }
    // the unused tail of every segment
    const int64_t n_thr = (int64_t)gridDim.x * blockDim.x;
    for (int64_t t = row; t < (int64_t)world * cap; t += n_thr) {
        const int d = (int)(t / cap);
        if (t - (int64_t)d * cap < s.seg[d]) continue;
        send[t * width + c_in] = -1.0f;
        pair_row[t] = -1;
        if (w) pair_w[t] = 0.0f;
    }
}

// The segments of a dispatch of no rows (B == 0, B_cap > 0): every slot lies past the pairs, filled as the tail of
// ep_scatter_kernel, so that the owners skip what this rank sends.
__global__ void ep_empty_kernel(int64_t n_slots, int width, int id_col, float* __restrict__ send, int* __restrict__ pair_row,
                                float* __restrict__ pair_w) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_slots) return;
    send[t * width + id_col] = -1.0f;
    pair_row[t] = -1;
    if (pair_w) pair_w[t] = 0.0f;
}

// out[row] = sum over the row's pairs in ascending sub-module order of back x w, from 0, multiply and add rounded separately
// (`out[rows[m]] += back[m] * w[m]`, mega_nerf.py:46-49); hard routing copies the row's one result.
__global__ void ep_combine_kernel(int64_t B, int K, const int* __restrict__ row_slots, const float* __restrict__ pair_w,
                                  const float* __restrict__ back, int out_cols, float* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * out_cols) return;
    const int64_t row = i / out_cols;
    const int c = (int)(i % out_cols);
    const float nan = __int_as_float(0x7fc00000);
    if (!pair_w) {
        const int slot = row_slots[row];
        out[i] = slot >= 0 ? back[(int64_t)slot * out_cols + c] : nan;
        return;
    }
    float acc = 0.0f;
    for (int k = 0; k < K; ++k) {
        const int slot = row_slots[row * K + k];
        if (slot >= 0) acc = __fadd_rn(acc, __fmul_rn(back[(int64_t)slot * out_cols + c], pair_w[slot]));
        else if (slot == -2) acc = nan;                          // dropped pair (segment overflow): poison, as combine_kernel
    }
    out[i] = acc;
}

// Backward of ep_combine_kernel: the gradient of every slot's result is its home row's gradient times the slot's blend weight
// (the gradient of `back[m] * w[m]`, one fp32 multiply), the row's gradient itself under hard routing, 0 past the pairs.
__global__ void ep_combine_backward_kernel(int64_t n_slots, const int* __restrict__ pair_row, const float* __restrict__ pair_w,
                                           const float* __restrict__ dout, int out_cols, float* __restrict__ dback) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_slots * out_cols) return;
    const int64_t slot = i / out_cols;
    const int c = (int)(i % out_cols);
    const int row = pair_row[slot];
    float g = 0.0f;
    if (row >= 0) {
        g = dout[(int64_t)row * out_cols + c];
        if (pair_w) g = __fmul_rn(g, pair_w[slot]);
    }
    dback[i] = g;
}

// Bucket counts of an owner call: the sub-module of each received row is given (payload column `id_col`, -1 = empty slot);
// the density noise column, if any, is copied to a contiguous [n] for the MLP kernels.
template <int KMAX>
__global__ void assigned_count_kernel(const float* __restrict__ rows, int64_t n, int stride, int id_col, int K, int64_t cap,
                                      int* counters, unsigned long long* __restrict__ mask_out, float* __restrict__ noise_out,
                                      unsigned int* status) {
    __shared__ int hist[MN_MAX_SUB];
    for (int i = threadIdx.x; i < K; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    const int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint64_t mask = 0;
    if (row < n) {
        const float id = rows[row * stride + id_col];
        if (id >= 0.0f) {
            const int k = (int)id;
            if (k < K && (float)k == id) mask = 1ull << k;
            else atomicOr(status, MN_STATUS_INDEX);
        }
        mask_out[row] = mask;
        if (noise_out) noise_out[row] = rows[row * stride + id_col + 1];
    }
    bucket_count<KMAX>(mask, K, cap, counters, hist);
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

size_t mn_route_assigned_scratch_bytes(int64_t n) {
    return mn_align((size_t)n * sizeof(unsigned long long)) + mn_align((size_t)n * sizeof(float));   // masks, density noise
}

int mn_route_build_assigned(mn_ctx* ctx, mn_model* m, const float* rows, int64_t n, int stride, int id_col, int has_noise, int64_t cap,
                            int* slot_row, void* scratch, const float** noise_out, cudaStream_t st) {
    unsigned long long* mask_buf = reinterpret_cast<unsigned long long*>(scratch);
    float* noise = has_noise ? reinterpret_cast<float*>(reinterpret_cast<char*>(scratch) + mn_align((size_t)n * sizeof(unsigned long long)))
                             : nullptr;
    *noise_out = noise;
    const int K = m->d.n_sub;
    MN_CUDA(ctx, cudaMemsetAsync(m->counters_d, 0, CNT_TOTAL * sizeof(int), st));
    MN_CUDA(ctx, cudaMemsetAsync(slot_row, 0xFF, (size_t)cap * sizeof(int), st));
    const unsigned blocks = (unsigned)mn_cdiv(n, 256);
    MN_ROUTE_DISPATCH(assigned_count_kernel, blocks, 256, rows, n, stride, id_col, K, cap, m->counters_d, mask_buf, noise, ctx->status_d);
    MN_LAUNCH_CHECK(ctx);
    MN_ROUTE_DISPATCH(route_scatter_kernel, blocks, 256, n, LiveRows{}, K, m->counters_d, cap, mask_buf, nullptr, slot_row, nullptr,
                      nullptr, ctx->status_d);
    MN_LAUNCH_CHECK(ctx);
    return MN_OK;
}

static size_t ep_scan_bytes(int64_t B, int K, int world, EpScan* s, void* base) {
    const int64_t blocks = mn_cdiv(B, EP_ROWS);
    size_t off = 0;
    auto take = [&](size_t n) { int* p = base ? (int*)((char*)base + off) : nullptr; off += mn_align(n); return p; };
    EpScan t{};
    t.blk = take((size_t)blocks * K * sizeof(int));
    t.start = take((size_t)K * sizeof(int));
    t.seg = take((size_t)world * sizeof(int));
    t.ticket = take(sizeof(int));
    if (s) *s = t;
    return off;
}

extern "C" {

int64_t mn_model_ep_segment_rows(const mn_model* m, int64_t B) {
    if (!m || B < 0) return 0;
    return B * (m->d.boundary_margin > 1.0f ? m->max_multiplicity : 1);
}

size_t mn_model_ep_dispatch_workspace_bytes(const mn_model* m, int64_t B, int world) {
    if (!m || B < 0 || world < 1) return 0;
    return ep_scan_bytes(B, m->d.n_sub, world, nullptr, nullptr);
}

int mn_model_ep_dispatch(mn_ctx* ctx, mn_model* m, const float* x_d, int64_t B, int64_t B_cap, int cols, const int32_t* assign_d,
                         const float* weights_d, const float* sigma_noise_d, int world, float* send_d, int32_t* counts_d,
                         int32_t* pair_row_d, float* pair_w_d, int32_t* row_slots_d, void* workspace_d, size_t workspace_bytes,
                         void* stream) {
    if (!ctx || !m || B < 0 || B_cap < B || world < 1) return MN_ERR_INVALID;
    if (m->d.kind != 2) return mn_fail(ctx, MN_ERR_INVALID, "mn_model_ep_dispatch: not a MegaNeRF model");
    const bool blend = m->d.boundary_margin > 1.0f;
    const int xoff = m->d.xyz_real ? 3 : 0;
    if (cols <= xoff) return mn_fail(ctx, MN_ERR_INVALID, "mn_model_ep_dispatch: rows have no child columns");
    const int64_t cap = mn_model_ep_segment_rows(m, B_cap);
    if (!counts_d || (cap > 0 && (!send_d || !pair_row_d || (blend && !pair_w_d))) ||
        (B > 0 && (!x_d || !row_slots_d || (blend ? !weights_d : !assign_d))))
        return mn_fail(ctx, MN_ERR_INVALID, "mn_model_ep_dispatch: missing buffer (weights / pair_w with boundary_margin > 1, else assign)");
    const int K = m->d.n_sub;
    cudaStream_t st = (cudaStream_t)stream;
    EpScan s;
    if (!workspace_d || workspace_bytes < ep_scan_bytes(B, K, world, &s, workspace_d))
        return mn_fail(ctx, MN_ERR_WORKSPACE, "mn_model_ep_dispatch: workspace too small");
    if (B == 0) {
        MN_CUDA(ctx, cudaMemsetAsync(counts_d, 0, (size_t)world * K * sizeof(int), st));
        if (cap == 0) return MN_OK;
        const int64_t n_slots = (int64_t)world * cap;
        const int c_in = cols - xoff;
        ep_empty_kernel<<<(unsigned)mn_cdiv(n_slots, 256), 256, 0, st>>>(n_slots, c_in + 1 + (sigma_noise_d ? 1 : 0), c_in, send_d,
                                                                        pair_row_d, blend ? pair_w_d : nullptr);
        MN_LAUNCH_CHECK(ctx);
        return MN_OK;
    }
    const float* w = blend ? weights_d : nullptr;
    const int* a = blend ? nullptr : assign_d;
    MN_CUDA(ctx, cudaMemsetAsync(s.ticket, 0, sizeof(int), st));
    const unsigned blocks = (unsigned)mn_cdiv(B, EP_ROWS);
    MN_ROUTE_DISPATCH(ep_count_kernel, blocks, EP_ROWS, a, w, B, K, world, s, counts_d);
    MN_LAUNCH_CHECK(ctx);
    MN_ROUTE_DISPATCH(ep_scatter_kernel, blocks, EP_ROWS, x_d, B, cols, xoff, a, w, sigma_noise_d, K, world, cap, s, send_d, pair_row_d,
                      blend ? pair_w_d : nullptr, row_slots_d, ctx->status_d);
    MN_LAUNCH_CHECK(ctx);
    return MN_OK;
}

int mn_model_ep_combine(mn_ctx* ctx, mn_model* m, int64_t B, const int32_t* row_slots_d, const float* pair_w_d, const float* back_d,
                        float* out_d, void* stream) {
    if (!ctx || !m || B < 0) return MN_ERR_INVALID;
    const bool blend = m->d.boundary_margin > 1.0f;
    if (B == 0) return MN_OK;
    if (!row_slots_d || !back_d || !out_d || (blend && !pair_w_d))
        return mn_fail(ctx, MN_ERR_INVALID, "mn_model_ep_combine: missing buffer");
    const int out_cols = m->nd.rgb_dim + 1;
    const int64_t n = B * out_cols;
    ep_combine_kernel<<<(unsigned)mn_cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(B, m->d.n_sub, row_slots_d, blend ? pair_w_d : nullptr,
                                                                                 back_d, out_cols, out_d);
    MN_LAUNCH_CHECK(ctx);
    return MN_OK;
}

int mn_model_ep_combine_backward(mn_ctx* ctx, mn_model* m, int64_t n_slots, const int32_t* pair_row_d, const float* pair_w_d,
                                 const float* dout_d, float* dback_d, void* stream) {
    if (!ctx || !m || n_slots < 0) return MN_ERR_INVALID;
    if (m->d.kind != 2) return mn_fail(ctx, MN_ERR_INVALID, "mn_model_ep_combine_backward: not a MegaNeRF model");
    const bool blend = m->d.boundary_margin > 1.0f;
    if (n_slots == 0) return MN_OK;
    if (!pair_row_d || !dout_d || !dback_d || (blend && !pair_w_d))
        return mn_fail(ctx, MN_ERR_INVALID, "mn_model_ep_combine_backward: missing buffer");
    const int out_cols = m->nd.rgb_dim + 1;
    const int64_t n = n_slots * out_cols;
    ep_combine_backward_kernel<<<(unsigned)mn_cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(n_slots, pair_row_d, blend ? pair_w_d : nullptr,
                                                                                          dout_d, out_cols, dback_d);
    MN_LAUNCH_CHECK(ctx);
    return MN_OK;
}

}  // extern "C"

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
