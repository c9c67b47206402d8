// Shared host/device definitions for libmn_b200.so.  The whole library is compiled with
// -fmad=false: every multiply-add that the fp32 oracle performs as two separately rounded torch ops
// stays two roundings here; fused multiply-adds appear only where written explicitly as fmaf().
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <string>

#include "../../include/mn_b200.h"

// device status bits (mn_ctx::status_d)
#define MN_STATUS_SPHERE 1u
#define MN_STATUS_OVERFLOW 2u
#define MN_STATUS_INDEX 4u

#include <vector>

// One element-wise re-layout of a weight tensor (fp32 transposes / sub-matrices / copies, fp16 tensor-core images).  The ~75 of
// them a sub-module needs are queued by mn_model_set_weights and run as TWO launches (fp32 layouts first, the fp16 images that read
// them second) instead of one tiny launch each: a training step re-packs every sub-module after the optimiser step.
enum { PK_COPY = 0, PK_TRANSPOSE, PK_SUBMATRIX, PK_TC_HALF, PK_TC_F32, PK_RGBW };
struct PackOp {
    const float* src;
    void* dst;
    void* dst2;
    long long count;
    int kind;
    int p[7];
};

struct mn_ctx {
    int device = 0;
    int sm_count = 132;
    std::string err;
    unsigned int* status_d = nullptr;
    long long launches = 0;             // kernels launched through this context (bench: gpu_launches)
    // optional CUDA-event timing of the MLP kernel launches (bench: roofline.achieved)
    int prof_on = 0;
    std::vector<cudaEvent_t> prof_ev;   // start/stop pairs
    size_t prof_used = 0;
    // queued weight re-layouts (see PackOp) and their device-side table
    std::vector<PackOp> pack_ops;
    PackOp* pack_ops_d = nullptr;
    size_t pack_ops_cap = 0;
};
void mn_pack_push(mn_ctx* ctx, const PackOp& op);
int mn_pack_flush(mn_ctx* ctx, cudaStream_t st);

static inline void mn_prof_begin(mn_ctx* ctx, cudaStream_t st) {
    if (!ctx->prof_on) return;
    if (ctx->prof_used + 2 > ctx->prof_ev.size()) {
        cudaEvent_t a, b;
        cudaEventCreate(&a);
        cudaEventCreate(&b);
        ctx->prof_ev.push_back(a);
        ctx->prof_ev.push_back(b);
    }
    cudaEventRecord(ctx->prof_ev[ctx->prof_used], st);
}
static inline void mn_prof_end(mn_ctx* ctx, cudaStream_t st) {
    if (!ctx->prof_on) return;
    cudaEventRecord(ctx->prof_ev[ctx->prof_used + 1], st);
    ctx->prof_used += 2;
}

static inline int mn_fail(mn_ctx* ctx, int code, const std::string& msg) {
    if (ctx) ctx->err = msg;
    return code;
}

#define MN_CUDA(ctx, expr)                                                                          \
    do {                                                                                            \
        cudaError_t _e = (expr);                                                                    \
        if (_e != cudaSuccess) {                                                                    \
            return mn_fail(ctx, MN_ERR_CUDA,                                                        \
                           std::string(#expr) + ": " + cudaGetErrorString(_e) + " (" + __FILE__ +   \
                               ":" + std::to_string(__LINE__) + ")");                               \
        }                                                                                           \
    } while (0)

#define MN_LAUNCH_CHECK(ctx)               \
    do {                                   \
        (ctx)->launches++;                 \
        MN_CUDA(ctx, cudaGetLastError());  \
    } while (0)

static inline int64_t mn_cdiv(int64_t a, int64_t b) { return (a + b - 1) / b; }
static inline size_t mn_align(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }

// ------------------------------------------------------------------------------------------------
// Where per-row network inputs come from (device-side view of mn_rows).
// ------------------------------------------------------------------------------------------------
struct RowSrc {
    const float* x;      // mode 0: [B, cols];  mode 1: xyz [B, cols]
    int cols;            // row stride of x
    int net_off;         // first network column inside x (3 when a real-xyz routing prefix is present)
    const float* dirs;   // per-ray (mode 1) or inside x (mode 0)
    int64_t dir_stride;
    const float* idx;
    int64_t idx_stride;
    int div;             // row -> ray divisor (1 in mode 0)
    int dir_quirk;       // models/nerf.py:146 x[:, -4:-1] with no index column: dir := (xyz_z, d_x, d_y)
    int xyz_dim;
    const int* gather;   // mode 1 only: row r reads sample gather[r] (the queried samples of an occupancy grid); NULL = row r

    __device__ __forceinline__ int64_t sample(int64_t row) const { return gather ? (int64_t)gather[row] : row; }
    __device__ __forceinline__ float xyz(int64_t row, int j) const { return x[sample(row) * cols + net_off + j]; }
    __device__ __forceinline__ float route_xyz(int64_t row, int j) const { return x[sample(row) * cols + j]; }
    __device__ __forceinline__ float dir(int64_t row, int j) const {
        const int64_t s = sample(row);
        if (dir_quirk) {
            // columns [-4:-1] of [xyz(3), dir(3)] are (z, d_x, d_y)
            if (j == 0) return x[s * cols + net_off + 2];
            return dirs[(s / div) * dir_stride + (j - 1)];
        }
        return dirs[(s / div) * dir_stride + j];
    }
    __device__ __forceinline__ float index(int64_t row) const { return idx[(sample(row) / div) * idx_stride]; }
};

// Rows of a call whose count lives on the device (the background pass of mn_render_rays_bg): `rays` points at a device count of
// live rays, each `mul` rows; rows at or past mul * *rays are not read or written.  rays == NULL: every one of the call's rows.
struct LiveRows {
    const int* rays;
    int mul;
    __device__ __forceinline__ int64_t rows(int64_t all) const { return rays ? (int64_t)*rays * mul : all; }
};

// ------------------------------------------------------------------------------------------------
// device helpers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float mn_pow2f(int k) { return __int_as_float((127 + k) << 23); }

// sin / cos of (2^k * x) exactly as the oracle evaluates them: the product is exact (power of two),
// then a full-range accurate sincos (no fast-math intrinsics).
__device__ __forceinline__ void mn_pe_sincos(float x, int k, float* s, float* c) {
    sincosf(x * mn_pow2f(k), s, c);
}

__device__ __forceinline__ float mn_softplus_shifted(float x) {
    // F.softplus(x - 1, beta=1, threshold=20)   (models/nerf.py:38-39)
    float y = x - 1.0f;
    return y > 20.0f ? y : log1pf(expf(y));
}

__device__ __forceinline__ float mn_sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }

__device__ __forceinline__ float mn_dot3(const float* a, const float* b) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }

// Depth at which ray [8] leaves the ellipsoid (center3, radius3; NULL radius = unit sphere at the origin), rendering.py:396-414.
// *outside: the closest point of the ray's line lies on or outside the surface (the camera is not bounded by it).
__device__ __forceinline__ float mn_sphere_far(const float* __restrict__ ray, const float* __restrict__ center,
                                               const float* __restrict__ radius, bool* outside) {
    float o[3], d[3];
    for (int j = 0; j < 3; ++j) {
        o[j] = ray[j];
        d[j] = ray[3 + j];
        if (radius) { o[j] = (o[j] - center[j]) / radius[j]; d[j] = d[j] / radius[j]; }
    }
    const float dd = mn_dot3(d, d);
    const float d1 = -mn_dot3(d, o) / dd;
    float p[3];
    for (int j = 0; j < 3; ++j) p[j] = o[j] + d1 * d[j];
    const float cosv = 1.0f / sqrtf(dd);
    const float pn2 = mn_dot3(p, p);
    *outside = pn2 >= 1.0f;
    return d1 + sqrtf(1.0f - pn2) * cosv;
}
