#pragma once

// Tensor-core MLP kernel for Hopper (sm_90a), included inside mn_mlp_tc.cu's anonymous namespace.
//
//   tc_mlp_wg_kernel<kMode, kSplit, kWide>   persistent, one 128-row tile at a time, 384 threads:
//     warpgroup 2     one thread streams the weight K-slabs of every GEMM (cp.async.bulk into an mbarrier ring) and the
//                     feature-tile segments (positional encodings, direction + appearance) into their own buffer
//     warpgroups 0-1  rows 0-63 / 64-127 of the tile: wgmma.mma_async m64nNk16 with A = the tile's fp16 activations (or the
//                     feature segment) in shared memory and B = the ring stage, fp32 accumulators in registers that start at
//                     the bias (PP_DGRAD: at 0); then the epilogue straight from the registers: ReLU -> fp16 -> the next
//                     layer's A operand, written IN PLACE (every MMA that read the old activations has completed), sigma and
//                     rgb heads -> HBM.
//   kMode == PP_INFER up to 256 wide without kSplit (wg_reg_act): each warpgroup keeps its activations in registers instead,
//   the A operand of the register form of wgmma, and the epilogue packs the accumulators straight into them.
//   The two consumer warpgroups share the weight stream (a ring stage is released when both have read it) and never touch
//   each other's rows.  GEMMs wider than 256 (the 512-wide network, kWide) run as two N = 256 halves; the first half's
//   fp16 result waits in registers until the second half has read the old activations.
//
//   kMode: PP_INFER (inference), PP_TRAIN_FWD (inference + every layer's fp16 activations and the head values written to the
//   training tapes), PP_DGRAD (the data-gradient chain of mn_train_tc.cuh on transposed weight images).
//   kSplit (tc_f16x3): three MMA passes per GEMM over hi / lo fp16 planes of both operands (hi*hi + hi*lo + lo*hi).
//
// Operand layout (see the top of mn_mlp_tc.cu): K-major, no swizzle, [K/8][rows][8] fp16.  wgmma descriptor: leading byte
// offset = rows * 16 (next 8 K-columns), stride byte offset = 128 (next 8 rows).

// wgmma.mma_async m64nNk16, fp16 operands from shared-memory descriptors, fp32 accumulators in registers (N/2 per thread).
// TA / TB: 0 = K-major operand, 1 = MN-major operand.  `accumulate` == 0 overwrites the accumulators.
template <int TA, int TB>
__device__ __forceinline__ void wg_mma_n16(float* d, uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, %11, %12;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wg_mma_n32(float* d, uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, %20;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wg_mma_n64(float* d, uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wg_mma_n128(float* d, uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %68;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wg_mma_n256(float* d, uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, %131, %132;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB));
}
template <int N, int TA = 0, int TB = 0>
__device__ __forceinline__ void wg_mma(float* d, uint64_t da, uint64_t db, uint32_t accumulate) {
    static_assert(N == 16 || N == 32 || N == 64 || N == 128 || N == 256, "wgmma N");
    if constexpr (N == 16) wg_mma_n16<TA, TB>(d, da, db, accumulate);
    else if constexpr (N == 32) wg_mma_n32<TA, TB>(d, da, db, accumulate);
    else if constexpr (N == 64) wg_mma_n64<TA, TB>(d, da, db, accumulate);
    else if constexpr (N == 128) wg_mma_n128<TA, TB>(d, da, db, accumulate);
    else wg_mma_n256<TA, TB>(d, da, db, accumulate);
}

// The same MMA with A from registers (the m64k16 fp16 fragment: a[0] / a[1] = rows ra / rb at columns 2 q4 + {0, 1}, a[2] /
// a[3] the same rows at columns 8 + 2 q4 + {0, 1}) and a K-major B from a shared-memory descriptor.
__device__ __forceinline__ void wg_mma_rs_n32(float* d, const uint32_t* a, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(accumulate));
}
__device__ __forceinline__ void wg_mma_rs_n64(float* d, const uint32_t* a, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(accumulate));
}
__device__ __forceinline__ void wg_mma_rs_n128(float* d, const uint32_t* a, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, p, 1, 1, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(accumulate));
}
__device__ __forceinline__ void wg_mma_rs_n256(float* d, const uint32_t* a, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %133, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, {%128, %129, %130, %131}, %132, p, 1, 1, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(accumulate));
}
template <int N>
__device__ __forceinline__ void wg_mma_rs(float* d, const uint32_t* a, uint64_t db, uint32_t accumulate) {
    static_assert(N == 32 || N == 64 || N == 128 || N == 256, "wgmma N");
    if constexpr (N == 32) wg_mma_rs_n32(d, a, db, accumulate);
    else if constexpr (N == 64) wg_mma_rs_n64(d, a, db, accumulate);
    else if constexpr (N == 128) wg_mma_rs_n128(d, a, db, accumulate);
    else wg_mma_rs_n256(d, a, db, accumulate);
}

__device__ __forceinline__ uint64_t wg_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)(lbo_bytes >> 4) << 16) | ((uint64_t)(sbo_bytes >> 4) << 32);
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void st_shared_u32(unsigned char* p, uint32_t v) { *reinterpret_cast<uint32_t*>(p) = v; }
// max(h, +0) on both halves of a packed fp16 pair (__hmax2: a NaN half gives +0, and max(-0, +0) = +0).  Rounding to fp16
// commutes with max(., 0), so relu_h2(pack_h2(a, b)) has the bits of pack_h2(fmaxf(a, 0.0f), fmaxf(b, 0.0f)) for every a, b.
__device__ __forceinline__ uint32_t relu_h2(uint32_t h) {
    const __half2 r = __hmax2(*reinterpret_cast<const __half2*>(&h), __float2half2_rn(0.0f));
    return *reinterpret_cast<const uint32_t*>(&r);
}
// Pins the accumulator registers at a point of the instruction stream (the compiler must not move reads or writes of them
// across it): placed after the accumulators are initialised and after the wait that completes the MMAs writing them.
template <int N>
__device__ __forceinline__ void wg_fence_operand(float* d) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// ---- the stage program: what every ring stage of one GEMM chunk (<= 256 output columns) carries.  The producer, both
// consumer warpgroups and the host-side test hook (mn_debug_tp_program) all walk it through wg_walk_chunk, so the roles
// agree on the ring traffic by construction.
enum { WS_FROM_X = 1, WS_X_FIRST = 2, WS_X_LAST = 4, WS_LO = 8, WS_CHUNK_FIRST = 16, WS_CHUNK_LAST = 32 };
struct WgStage {
    int w_off;       // byte offset of the weight slab inside the sub-module's pack (lo plane included for pass 1)
    int w_bytes;     // kc * nw * 2
    int nw;          // rows of the slab = B operand N (min(N, 256))
    int kc;          // K columns of the slab (multiple of 16, <= slab)
    int a_col;       // first K column of the A operand: in the activation buffer, or in the feature segment (WS_FROM_X)
    int x_off;       // WS_X_FIRST: byte offset of the feature segment inside the tile's feature record (one plane)
    int x_bytes;     // WS_X_FIRST: bytes of that segment
    int flags;       // WS_*: WS_LO = pass 2 (A operand and features from the lo planes)
};
template <class F>
__host__ __device__ __forceinline__ void wg_walk_chunk(const TcPlan& P, int gi, int ch, int npass, int slab, F&& f) {
    const TcGemm& g = P.g[gi];
    const int nw = g.n < 256 ? g.n : 256, ktot = g.k[0] + (g.nseg > 1 ? g.k[1] : 0);
    int first = WS_CHUNK_FIRST;
    for (int pass = 0; pass < npass; ++pass) {
        // pass 0: A_hi * W_hi, pass 1: A_hi * W_lo, pass 2: A_lo * W_hi.  Weight image of a GEMM: [N/256 halves][K/8][min(N, 256)][8]
        const int wbase = (pass == 1 ? P.plane_bytes : 0) + g.w_off + ch * ktot * nw * 2;
        int kbase = 0;
        for (int sgi = 0; sgi < g.nseg; ++sgi) {
            const int kseg = g.k[sgi];
            const bool fx = g.src[sgi] != SRC_H;
            for (int k0 = 0; k0 < kseg; k0 += slab) {
                WgStage st;
                st.kc = kseg - k0 < slab ? kseg - k0 : slab;
                st.nw = nw;
                st.w_off = wbase + (kbase + k0) * nw * 2;
                st.w_bytes = st.kc * nw * 2;
                st.a_col = k0;
                st.x_off = fx && k0 == 0 ? (g.src[sgi] == SRC_XAUX ? P.kpe * kTileM * 2 : 0) : 0;
                st.x_bytes = fx && k0 == 0 ? kseg * kTileM * 2 : 0;
                const bool last = pass == npass - 1 && sgi == g.nseg - 1 && k0 + slab >= kseg;
                st.flags = first | (fx ? WS_FROM_X : 0) | (fx && k0 == 0 ? WS_X_FIRST : 0) | (fx && k0 + slab >= kseg ? WS_X_LAST : 0) |
                           (pass == 2 ? WS_LO : 0) | (last ? WS_CHUNK_LAST : 0);
                first = 0;
                f(st);
            }
            kbase += kseg;
        }
    }
}

// Three full warpgroups: two consumers and the producer warpgroup (one of its threads issues the copies).  The launch alone caps
// every thread at 168 registers (65536 / 384, rounded down); setmaxnreg then moves registers from the producer warpgroup
// (kWgProducerRegs) to the consumers (kWgConsumerRegs): 128 x 56 + 256 x 224 = 64512 <= 65536.  The producer's stage walk
// spills below 56 registers; with 224 per consumer thread only the 512-wide variant still spills.
constexpr int kWgmmaThreads = 384;
constexpr int kWgProducerRegs = 56;
constexpr int kWgConsumerRegs = 224;
constexpr int kWgRingMax = 8;

struct WgLayout {
    int ring, h, xa, f32, f32_vec4, dsig, bars, total, stages, slab, stage_bytes;
};

// Whether a variant keeps each consumer warpgroup's activations in registers, as the A operand of the register form of wgmma,
// instead of in the shared tile image Hs: the tc_f16 inference kernel up to 256 wide.  The training variants write every
// layer's image to the tapes from Hs, tc_f16x3 needs hi and lo planes, and the 512-wide activations do not fit in registers.
__host__ __device__ constexpr bool wg_reg_act(int mode, bool split, bool wide) { return mode == PP_INFER && !split && !wide; }

// ring first: an MMA of a narrow GEMM rounded up to the next supported N reads (and ignores) up to 512 bytes past its stage.
// reg_act (wg_reg_act): no Hs region, the ring takes its place.
__host__ __device__ inline WgLayout wg_layout(const TcPlan& p, bool split, bool reg_act) {
    WgLayout s;
    const int kx = p.kpe > p.kaux ? p.kpe : p.kaux;
    const int nw = p.L > 256 ? 256 : p.L;                   // widest B slab (no GEMM is wider than layer_dim)
    const int h_bytes = reg_act ? 0 : p.L * kTileM * 2 * (split ? 2 : 1);
    s.slab = (split || p.L > 256) ? 32 : 64;
    s.stage_bytes = s.slab * nw * 2;
    s.f32_vec4 = (p.f32_floats + 3) / 4;
    const int fixed = h_bytes + kx * kTileM * 2 + s.f32_vec4 * 16 + kTileM * 4 + 256;
    int st = (kSmemMax - fixed) / s.stage_bytes;
    if (st > kWgRingMax) st = kWgRingMax;
    s.stages = st;
    s.ring = 0;
    s.h = st * s.stage_bytes;
    s.xa = s.h + h_bytes;
    s.f32 = s.xa + kx * kTileM * 2;
    s.dsig = s.f32 + s.f32_vec4 * 16;
    s.bars = s.dsig + kTileM * 4;
    s.total = s.bars + 256;
    return s;
}

// ---- head stage of the data-gradient chain (nerf.py:132-160 backwards), per row; shared by tc_mlp_wg_kernel<PP_DGRAD> and the
// layer-GEMM path's tc_layer_head_dgrad_kernel.
// d[c] = gradient of the rgb Linear's output c: upstream gradient x blend weight, then sigmoid' (colour head, rgb_dim 3) or the
// raw SH coefficients as they are.  Returns the gradient of the sigma pre-activation (softplus' or ReLU').  tf: the row's entry
// of the tape's fp32 head block.  kR bounds rgb_dim (d holds kR floats).  Only compile-time indices into d (loops unrolled to
// kR and left at c == R), so the array stays in registers.
template <int kR>
__device__ __forceinline__ float tc_head_grad(const MlpArgs& m, const float* grad_out, int64_t row, int64_t slot, const float* tf,
                                              float* d) {
    const int R = m.nd.rgb_dim;
    float gsig = 0.0f;
    if (R == 3) {
        float g0 = 0.0f, g1 = 0.0f, g2 = 0.0f;
        if (row >= 0) {
            const float4 gv = *reinterpret_cast<const float4*>(grad_out + row * 4);
            const float bw = m.slot_w ? m.slot_w[slot] : 1.0f;
            g0 = gv.x * bw; g1 = gv.y * bw; g2 = gv.z * bw; gsig = gv.w * bw;
        }
        const float c0v = tf[MN_TC_F32_RGB * kTileM], c1v = tf[(MN_TC_F32_RGB + 1) * kTileM], c2v = tf[(MN_TC_F32_RGB + 2) * kTileM];
        d[0] = (g0 * (1.0f - c0v)) * c0v; d[1] = (g1 * (1.0f - c1v)) * c1v; d[2] = (g2 * (1.0f - c2v)) * c2v;
    } else {
#pragma unroll
        for (int c = 0; c < kR; ++c) d[c] = 0.0f;
        if (row >= 0) {
            const float* go = grad_out + row * m.out_cols;          // [rgb_dim SH coefficients][sigma]
            const float bw = m.slot_w ? m.slot_w[slot] : 1.0f;
#pragma unroll
            for (int c = 0; c < kR; ++c) {
                if (c >= R) break;
                d[c] = go[c] * bw;
            }
            gsig = go[R] * bw;
        }
    }
    const float pre = tf[MN_TC_F32_SIGMA * kTileM];
    float dsp;
    if (m.nd.softplus) { const float y = pre - 1.0f; dsp = y > 20.0f ? 1.0f : 1.0f / (1.0f + expf(-y)); }
    else dsp = pre > 0.0f ? 1.0f : 0.0f;
    return gsig * dsp;
}

// v[e] = mask(G > 0) (sum_c W_rgb[c][k0 + e] d[c]) for the 8 columns k0 .. k0 + 7 of one row; Wr = [rgb_dim][half] fp32, g = the
// row's 8 fp16 values of G in the tile image, d = kR floats (tc_head_grad).  Order c = 0, 1, .. (a product, then one fma per
// further row).
template <int kR>
__device__ __forceinline__ void tc_rgb_dgrad8(const float* Wr, int half, int k0, const float* d, int R, const unsigned char* g, float* v) {
    const uint4 gm = *reinterpret_cast<const uint4*>(g);
    const __half2* gh = reinterpret_cast<const __half2*>(&gm);
    {
        const float4 wa = *reinterpret_cast<const float4*>(Wr + k0), wb = *reinterpret_cast<const float4*>(Wr + k0 + 4);
        v[0] = wa.x * d[0]; v[1] = wa.y * d[0]; v[2] = wa.z * d[0]; v[3] = wa.w * d[0];
        v[4] = wb.x * d[0]; v[5] = wb.y * d[0]; v[6] = wb.z * d[0]; v[7] = wb.w * d[0];
    }
#pragma unroll
    for (int c = 1; c < kR; ++c) {
        if (c >= R) break;
        const float4 wa = *reinterpret_cast<const float4*>(Wr + c * half + k0);
        const float4 wb = *reinterpret_cast<const float4*>(Wr + c * half + k0 + 4);
        v[0] = fmaf(wa.x, d[c], v[0]); v[1] = fmaf(wa.y, d[c], v[1]); v[2] = fmaf(wa.z, d[c], v[2]); v[3] = fmaf(wa.w, d[c], v[3]);
        v[4] = fmaf(wb.x, d[c], v[4]); v[5] = fmaf(wb.y, d[c], v[5]); v[6] = fmaf(wb.z, d[c], v[6]); v[7] = fmaf(wb.w, d[c], v[7]);
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) {
        const float gv = (e & 1) ? __high2float(gh[e >> 1]) : __low2float(gh[e >> 1]);
        v[e] = gv > 0.0f ? v[e] : 0.0f;
    }
}

// Appearance-embedding gradient, step 1: per-image sums of dZ_dira rows (fp32, unscaled).  Called by a whole warp; the lanes
// are consecutive slots, i.e. mostly samples of one ray = one image id.  sums = column k0 of image 0 of the sub-module's
// [app_count][half] block.
__device__ __forceinline__ void tc_emb_sums8(float* sums, int half, bool valid, int id, int lane, const float* v) {
    unsigned todo = __ballot_sync(0xffffffffu, valid);
    while (todo) {
        const int leader = __ffs(todo) - 1;
        const int cur = __shfl_sync(0xffffffffu, id, leader);
        const bool mine = valid && id == cur;
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            float s = mine ? v[e] : 0.0f;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if (lane == leader) atomicAdd(sums + (size_t)cur * half + e, s);
        }
        todo &= ~__ballot_sync(0xffffffffu, mine);
    }
}

template <int kMode, bool kSplit, bool kWide>
__global__ void __launch_bounds__(kWgmmaThreads, 1) tc_mlp_wg_kernel(const TcArgs A) {
    extern __shared__ __align__(1024) unsigned char smem[];
    constexpr bool kRegAct = wg_reg_act(kMode, kSplit, kWide);
    const TcPlan& P = A.plan;
    const WgLayout SL = wg_layout(P, kSplit, kRegAct);
    const int stages = SL.stages, slab = SL.slab, stage_bytes = SL.stage_bytes;
    unsigned char* ring = smem + SL.ring;
    unsigned char* Hs = smem + SL.h;
    unsigned char* XA = smem + SL.xa;
    float* F32 = reinterpret_cast<float*>(smem + SL.f32);        // fp32 block (biases, sigma weights) of the current sub-module
    float* DSIG = reinterpret_cast<float*>(smem + SL.dsig);      // PP_DGRAD: S * d(sigma pre-activation) per tile row
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + SL.bars);
    uint64_t* full = bars;                   // [kWgRingMax]
    uint64_t* empty = bars + kWgRingMax;     // [kWgRingMax], one arrival per consumer warpgroup
    uint64_t* xa_full = bars + 2 * kWgRingMax;
    uint64_t* xa_empty = xa_full + 1;

    const int n_gemm = A.m.sigma_only ? P.n_trunk : P.n_gemm;
    constexpr int npass = kSplit ? 3 : 1;

    if (threadIdx.x == 0) {
        for (int i = 0; i < kWgRingMax; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 2); }
        mbar_init(xa_full, 1);
        mbar_init(xa_empty, 2);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    const int wgi = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 7), 0);     // warp-uniform role
    if (wgi == 2) {
        // =========================== producer ===========================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kWgProducerRegs));
        if (threadIdx.x == 256) {
            // the tile count is computed by each role after setmaxnreg: carried across the role split, ptxas spilled it
            const int64_t n_tiles = (A.m.n_slots() + kTileM - 1) / kTileM;
            int stage = 0;
            uint32_t phase = 0, xphase = 0;
            const int64_t xtile_bytes = (int64_t)(P.kpe + P.kaux) * kTileM * 2;
            for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
                const unsigned char* wsub = A.wpack + (size_t)A.m.sub_of_tile(tile) * P.sub_bytes;
                const unsigned char* xtile = reinterpret_cast<const unsigned char*>(A.ximg) + tile * xtile_bytes;
                for (int gi = 0; gi < n_gemm; ++gi) {
                    const int nch = (P.g[gi].n + 255) >> 8;
                    for (int ch = 0; ch < nch; ++ch) {
                        wg_walk_chunk(P, gi, ch, npass, slab, [&](const WgStage& st) {
                            if (st.flags & WS_X_FIRST) {
                                mbar_wait(xa_empty, xphase ^ 1);
                                mbar_expect_tx(xa_full, (uint32_t)st.x_bytes);
                                bulk_g2s(XA, xtile + ((st.flags & WS_LO) ? A.x_plane_halves * 2 : 0) + st.x_off, (uint32_t)st.x_bytes, xa_full);
                                xphase ^= 1;
                            }
                            mbar_wait(&empty[stage], phase ^ 1);
                            mbar_expect_tx(&full[stage], (uint32_t)st.w_bytes);
                            bulk_g2s(ring + (size_t)stage * stage_bytes, wsub + st.w_off, (uint32_t)st.w_bytes, &full[stage]);
                            if (++stage == stages) { stage = 0; phase ^= 1; }
                        });
                    }
                }
            }
        }
    } else {
        // =========================== consumers: MMA + epilogue ===========================
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kWgConsumerRegs));
        const int64_t n_slots = A.m.n_slots();
        const int64_t n_tiles = (n_slots + kTileM - 1) / kTileM;
        const int wg = wgi;
        const int t = threadIdx.x & 127, w = t >> 5, lane = t & 31, q4 = lane & 3;
        // accumulator fragment of m64nNk16: this thread holds rows ra, ra + 8 and, in every 8-column group j, columns 8j + 2 q4 + {0, 1}
        const int ra = 64 * wg + 16 * w + (lane >> 2), rb = ra + 8;
        const uint32_t ring_s = smem_u32(ring), h_s = smem_u32(Hs), xa_s = smem_u32(XA);
        const uint32_t row_base = (uint32_t)(64 * wg * 16);
        const int L = P.L;
        const uint32_t lo_bytes = (uint32_t)(L * kTileM * 2);
        const uint32_t bar_id = 1 + wg;
        auto wg_sync = [&]() { asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory"); };
        int stage = 0, cur_sub = -1;
        uint32_t phase = 0, xphase = 0;
        // kRegAct: this warpgroup's rows of the previous GEMM's fp16 output, 4 registers per 16 K-columns (the m64k16 A fragment,
        // which has the accumulator fragment's row / column map: hreg[2 j] / hreg[2 j + 1] = rows ra / rb, column group j)
        uint32_t hreg[kRegAct ? 64 : 1];

        for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
            const int sub = A.m.sub_of_tile(tile);
            if (sub != cur_sub) {
                // both warpgroups stage the sub-module's fp32 block (it changes a handful of times per launch): epilogue
                // operands from shared memory instead of dependent global loads between the activation stores
                asm volatile("bar.sync 3, 256;" ::: "memory");
                const float4* src = reinterpret_cast<const float4*>(A.wpack + (size_t)sub * P.sub_bytes + P.f32_off);
                for (int i = threadIdx.x; i < SL.f32_vec4; i += 256) reinterpret_cast<float4*>(F32)[i] = src[i];
                asm volatile("bar.sync 3, 256;" ::: "memory");
                cur_sub = sub;
            }
            const int64_t slot_a = tile * kTileM + ra, slot_b = tile * kTileM + rb;
            const int64_t row_a = A.m.row_of_slot(slot_a, n_slots), row_b = A.m.row_of_slot(slot_b, n_slots);
            float sig_a = 0.0f, sig_b = 0.0f;

            if (kMode == PP_DGRAD) {
                // ---- head stage of the data-gradient chain (nerf.py:132-160 backwards): upstream gradient x blend weight ->
                // sigmoid' (colour head, rgb_dim 3; raw SH coefficients pass through) / softplus' -> rgb Linear transposed
                // (rgb_dim -> L/2, CUDA cores) -> ReLU mask of dir_a_encoding -> dZ_dira as the first A operand (columns
                // 0 .. L/2-1 of the activation buffer) and on the gradient tape; per-image sums of its rows for the
                // appearance-embedding gradient; head pre-activation gradients in fp32 for their own Linears.
                // Thread t of the warpgroup: row 64 wg + t % 64, column half t / 64 (the lanes of a warp are 32 consecutive rows).
                const float S = *A.scale;
                const int hr = 64 * wg + (t & 63), part = t >> 6;
                const int64_t hslot = tile * kTileM + hr;
                const int64_t hrow = A.m.row_of_slot(hslot, n_slots);
                const int R = A.m.nd.rgb_dim;
                const float* Wr = F32 + L;                                  // [rgb_dim][L/2] rgb weights (fp32 block of the data-gradient plan)
                const float* tf = A.tape_f32 + (size_t)tile * MN_TC_F32_ROWS * kTileM + hr;
                float d[MN_TC_RGB_MAX];
                const float ds = tc_head_grad<MN_TC_RGB_MAX>(A.m, A.grad_out, hrow, hslot, tf, d);
                if (part == 0) {
                    DSIG[hr] = ds * S;
                    float* tg = A.tape_gf32 + (size_t)tile * mn_tc_g32_rows(R) * kTileM + hr;
                    tg[MN_TC_G32_SIGMA * kTileM] = ds;
#pragma unroll
                    for (int c = 0; c < MN_TC_RGB_MAX; ++c) {
                        if (c >= R) break;
                        tg[(MN_TC_G32_RGB + c) * kTileM] = d[c];
                    }
                }
                const int id = (int)tf[MN_TC_F32_ID * kTileM];
                const unsigned char* gimg = A.tape_act + (size_t)tile * A.act_tile_bytes + mn_tc_img_off(A.layers + 1, L);
                unsigned char* dimg = A.tape_dz + (size_t)tile * A.act_tile_bytes + mn_tc_img_off(A.layers + 1, L);
                const int half = L / 2, per = half / 2;
                for (int kk = 0; kk < per; kk += 8) {
                    const int k0 = part * per + kk;
                    float v[8];
                    tc_rgb_dgrad8<MN_TC_RGB_MAX>(Wr, half, k0, d, R, gimg + (size_t)(k0 >> 3) * (kTileM * 16) + (size_t)hr * 16, v);
                    if (A.emb_sum) tc_emb_sums8(A.emb_sum + (size_t)sub * A.m.nd.app_count * half + k0, half, hrow >= 0, id, lane, v);
                    uint32_t pk[4];
#pragma unroll
                    for (int e = 0; e < 4; ++e) pk[e] = pack_h2(v[2 * e] * S, v[2 * e + 1] * S);
                    const uint4 outv = make_uint4(pk[0], pk[1], pk[2], pk[3]);
                    *reinterpret_cast<uint4*>(Hs + (size_t)(k0 >> 3) * (kTileM * 16) + (size_t)hr * 16) = outv;
                    *reinterpret_cast<uint4*>(dimg + (size_t)(k0 >> 3) * (kTileM * 16) + (size_t)hr * 16) = outv;
                }
                fence_proxy_async();
                wg_sync();
            }

            for (int gi = 0; gi < n_gemm; ++gi) {
                const TcGemm& gm = P.g[gi];
                auto gemm = [&](auto nm_tag) {
                    constexpr int NM = decltype(nm_tag)::value;        // MMA N (gm.n rounded up; extra columns are ignored)
                    float acc[NM / 2];
                    uint32_t held[kWide ? NM / 4 : 1];
                    const int nch = (gm.n + 255) >> 8;
                    const bool rgb = gm.epi == EPI_RGB;
                    const bool want_sigma = gm.epi == EPI_RELU_SIGMA;
                    const bool publish = !(want_sigma && A.m.sigma_only);   // nobody reads H after the last trunk layer
                    const float* sw = F32 + P.sigma_w_off;
                    float sacc_a = 0.0f, sacc_b = 0.0f;
                    // every forward GEMM, rgb included, starts its accumulators at the bias (wgmma computes D = A B + D), so no
                    // epilogue adds one; the data-gradient chain starts at 0.  A compile-time choice: accumulators defined by
                    // a run-time choice of the two (zero for rgb only) make ptxas serialise the wgmma pipeline (C7515).
                    constexpr bool biased = kMode != PP_DGRAD;
                    for (int ch = 0; ch < nch; ++ch) {
                        if constexpr (biased) {
                            // rows ra and rb take column c's bias: acc[4 j .. 4 j + 3] = (ra, c), (ra, c + 1), (rb, c), (rb, c + 1).
                            // Columns past gm.n start at whatever follows the bias in shared memory; nothing reads them.
                            const float* bias = F32 + gm.bias_off + ch * 256;
#pragma unroll
                            for (int j = 0; j < NM / 8; ++j) {
                                const float2 bv = *reinterpret_cast<const float2*>(bias + 8 * j + 2 * q4);
                                acc[4 * j] = bv.x; acc[4 * j + 1] = bv.y; acc[4 * j + 2] = bv.x; acc[4 * j + 3] = bv.y;
                            }
                        } else {
#pragma unroll
                            for (int i = 0; i < NM / 2; ++i) acc[i] = 0.0f;
                        }
                        wg_fence_operand<NM / 2>(acc);
                        int prev = -1;
                        uint32_t accum = biased ? 1u : 0u;
                        wg_walk_chunk(P, gi, ch, npass, slab, [&](const WgStage& st) {
                            const bool from_x = (st.flags & WS_FROM_X) != 0;
                            // lo plane of H lives right after the hi plane (split mode); the feature buffer is reloaded per pass
                            const uint32_t a_base = (from_x ? xa_s : h_s + ((st.flags & WS_LO) ? lo_bytes : 0u)) + row_base;
                            if (st.flags & WS_X_FIRST) { mbar_wait(xa_full, xphase); xphase ^= 1; }
                            mbar_wait(&full[stage], phase);
                            const uint32_t b_base = ring_s + (uint32_t)(stage * stage_bytes);
                            wg_fence();
                            auto mma_smem_a = [&]() {
                                for (int kk = 0; kk < st.kc; kk += 16) {
                                    const uint64_t ad = wg_desc(a_base + (uint32_t)((st.a_col + kk) >> 3) * (kTileM * 16), kTileM * 16, 128);
                                    const uint64_t bd = wg_desc(b_base + (uint32_t)((kk >> 3) * st.nw * 16), (uint32_t)st.nw * 16, 128);
                                    wg_mma<NM>(acc, ad, bd, accum);
                                    accum = 1;
                                }
                            };
                            if constexpr (kRegAct) {
                                if (from_x) mma_smem_a();
                                else {
                                    // K-steps a_col / 16 .. (a_col + kc) / 16 - 1 of the activations: one branch per K-step keeps
                                    // every register index a compile-time constant
                                    const int k0 = st.a_col >> 4, k1 = (st.a_col + st.kc) >> 4;
#pragma unroll
                                    for (int k = 0; k < 16; ++k) {
                                        if (k < k0 || k >= k1) continue;
                                        const uint64_t bd = wg_desc(b_base + (uint32_t)(2 * (k - k0) * st.nw * 16), (uint32_t)st.nw * 16, 128);
                                        wg_mma_rs<NM>(acc, hreg + 4 * k, bd, accum);
                                        accum = 1;
                                    }
                                }
                            } else {
                                mma_smem_a();
                            }
                            wg_commit();
                            // the MMAs of the previous stage have completed: release it (one arrival per warpgroup)
                            if (prev >= 0) {
                                wg_wait<1>();
                                if (t == 0) mbar_arrive(&empty[prev]);
                            }
                            prev = stage;
                            if (++stage == stages) { stage = 0; phase ^= 1; }
                            if (st.flags & WS_X_LAST) {
                                wg_wait<0>();
                                if (t == 0) { mbar_arrive(&empty[prev]); mbar_arrive(xa_empty); }
                                prev = -1;
                            }
                        });
                        wg_wait<0>();
                        wg_fence_operand<NM / 2>(acc);
                        if (prev >= 0 && t == 0) mbar_arrive(&empty[prev]);
                        if (!kRegAct) wg_sync();     // every warp's MMAs have read the old activations: the epilogue may overwrite them

                        const int cb = ch * 256;
                        if (kMode == PP_DGRAD) {
                            // dH = accumulator (scaled by S) [+ S dsigma x w_sigma] -> ReLU mask from the activation tape -> fp16 ->
                            // next A operand + gradient tape.  The mask image and the target image coincide: dZ_l = dH_l where H_l > 0.
                            // N = 512 (kWide): chunk 0 (columns 0..255) goes to the gradient tape at once, but its fp16 pairs wait in
                            // `held` until chunk 1's MMAs have read the old dZ from Hs.
                            const size_t ioff = (size_t)tile * A.act_tile_bytes + mn_tc_img_off(gm.img, L);
                            const unsigned char* mimg = A.tape_act + ioff;
                            unsigned char* dimg = A.tape_dz + ioff;
                            const float dsa = DSIG[ra], dsb = DSIG[rb];
                            const int c0 = kWide ? cb : 0;
                            const bool dhold = kWide && nch == 2 && ch == 0;
                            constexpr int JB = NM / 8 < 8 ? NM / 8 : 8;        // column groups whose loads are issued together
#pragma unroll
                            for (int j0 = 0; j0 < NM / 8; j0 += JB) {
                            __half2 mka[JB], mkb[JB];
#pragma unroll
                            for (int jj = 0; jj < JB; ++jj) {
                                const int c = c0 + 8 * (j0 + jj) + 2 * q4;
                                const size_t po = (size_t)(c >> 3) * (kTileM * 16) + (size_t)ra * 16 + (size_t)(c & 7) * 2;
                                mka[jj] = mkb[jj] = __float2half2_rn(1.0f);
                                if (gm.epi != EPI_D_LINEAR && c0 + 8 * (j0 + jj) < gm.n) {
                                    mka[jj] = *reinterpret_cast<const __half2*>(mimg + po);
                                    mkb[jj] = *reinterpret_cast<const __half2*>(mimg + po + 128);
                                }
                            }
#pragma unroll
                            for (int jj = 0; jj < JB; ++jj) {
                                const int j = j0 + jj;
                                const int c = c0 + 8 * j + 2 * q4;
                                if (c0 + 8 * j >= gm.n) continue;
                                float a0 = acc[4 * j], a1 = acc[4 * j + 1], b0 = acc[4 * j + 2], b1 = acc[4 * j + 3];
                                if (gm.epi == EPI_D_MASK_SIGMA) {                                      // F32[0..L) = sigma weights
                                    const float2 s = *reinterpret_cast<const float2*>(F32 + c);
                                    a0 = fmaf(dsa, s.x, a0); a1 = fmaf(dsa, s.y, a1);
                                    b0 = fmaf(dsb, s.x, b0); b1 = fmaf(dsb, s.y, b1);
                                }
                                const size_t po = (size_t)(c >> 3) * (kTileM * 16) + (size_t)ra * 16 + (size_t)(c & 7) * 2;
                                if (gm.epi != EPI_D_LINEAR) {
                                    const __half2 ma = mka[jj], mb = mkb[jj];
                                    if (!(__low2float(ma) > 0.0f)) a0 = 0.0f;
                                    if (!(__high2float(ma) > 0.0f)) a1 = 0.0f;
                                    if (!(__low2float(mb) > 0.0f)) b0 = 0.0f;
                                    if (!(__high2float(mb) > 0.0f)) b1 = 0.0f;
                                }
                                const uint32_t ha = pack_h2(a0, a1), hb = pack_h2(b0, b1);
                                if (dhold) {
                                    held[(2 * j) % (NM / 4)] = ha;
                                    held[(2 * j + 1) % (NM / 4)] = hb;
                                } else {
                                    st_shared_u32(Hs + po, ha);
                                    st_shared_u32(Hs + po + 128, hb);
                                }
                                *reinterpret_cast<uint32_t*>(dimg + po) = ha;
                                *reinterpret_cast<uint32_t*>(dimg + po + 128) = hb;
                            }
                            }
                            if (kWide && nch == 2 && ch == 1) {
#pragma unroll
                                for (int j = 0; j < NM / 8; ++j) {
                                    const int c = 8 * j + 2 * q4;
                                    const size_t po = (size_t)(c >> 3) * (kTileM * 16) + (size_t)ra * 16 + (size_t)(c & 7) * 2;
                                    st_shared_u32(Hs + po, held[(2 * j) % (NM / 4)]);
                                    st_shared_u32(Hs + po + 128, held[(2 * j + 1) % (NM / 4)]);
                                }
                            }
                            fence_proxy_async();
                            wg_sync();
                            continue;
                        }
                        if (rgb) {
                            // rgb head: the 4 lanes of a quad hold a row's 32 columns (bias included); gather them into one lane per row
                            uint32_t va[32], vb[32];
#pragma unroll
                            for (int c = 0; c < 32; ++c) {
                                const int src = (lane & ~3) | ((c & 7) >> 1);
                                va[c] = __shfl_sync(0xffffffffu, __float_as_uint(acc[(4 * (c >> 3) + (c & 1)) % (NM / 2)]), src);
                                vb[c] = __shfl_sync(0xffffffffu, __float_as_uint(acc[(4 * (c >> 3) + 2 + (c & 1)) % (NM / 2)]), src);
                            }
                            if (q4 < 2) {
                                const int r = q4 ? rb : ra;
                                const int64_t row = q4 ? row_b : row_a, slot = q4 ? slot_b : slot_a;
                                float* tr = kMode == PP_TRAIN_FWD ? A.tape_f32 + (size_t)tile * MN_TC_F32_ROWS * kTileM + MN_TC_F32_RGB * kTileM + r : nullptr;
                                if (row >= 0) tc_emit_rgb(A.m, A.m.nd.affine ? sub : 0, row, slot, q4 ? vb : va, nullptr, q4 ? sig_b : sig_a, tr);
                                else if (tr) { tr[0] = 0.5f; tr[kTileM] = 0.5f; tr[2 * kTileM] = 0.5f; }
                            }
                            continue;
                        }
                        // training forward: tape image of this GEMM's output (trunk layer gi; then F, then G)
                        unsigned char* timg = kMode == PP_TRAIN_FWD ? A.tape_act + (size_t)tile * A.act_tile_bytes + mn_tc_img_off(gi, L) : nullptr;
                        const bool relu = gm.epi != EPI_LINEAR;
                        [[maybe_unused]] const bool hold = kWide && nch == 2 && ch == 0;
                        auto put = [&](int cc, uint32_t ha, uint32_t hb, float a0, float a1, float b0, float b1) {
                            const size_t po = (size_t)(cc >> 3) * (kTileM * 16) + (size_t)ra * 16 + (size_t)(cc & 7) * 2;
                            st_shared_u32(Hs + po, ha);
                            st_shared_u32(Hs + po + 128, hb);
                            if (kSplit) {
                                const float2 fa = __half22float2(*reinterpret_cast<const __half2*>(&ha));
                                const float2 fb = __half22float2(*reinterpret_cast<const __half2*>(&hb));
                                st_shared_u32(Hs + lo_bytes + po, pack_h2(a0 - fa.x, a1 - fa.y));
                                st_shared_u32(Hs + lo_bytes + po + 128, pack_h2(b0 - fb.x, b1 - fb.y));
                            }
                            if (timg) {
                                *reinterpret_cast<uint32_t*>(timg + po) = ha;
                                *reinterpret_cast<uint32_t*>(timg + po + 128) = hb;
                            }
                        };
                        constexpr int JB = NM / 8 < 8 ? NM / 8 : 8;            // column groups whose loads are issued together
                        if constexpr (kRegAct) {
                            // kHR: a ReLU layer without the sigma head, the ReLU on the packed fp16 pairs.  Its own copy of the
                            // loop leaves no fp32 ReLU or sigma instructions for the compiler to predicate off: they would
                            // still be issued.  Every column group is written, so no register keeps its old value across the
                            // epilogue; groups past gm.n hold values that no MMA reads (the next K is at most gm.n).
                            auto epi = [&](auto hr_tag) {
                                constexpr bool kHR = decltype(hr_tag)::value;
#pragma unroll
                                for (int j0 = 0; j0 < NM / 8; j0 += JB) {
                                    float2 svs[JB];
#pragma unroll
                                    for (int jj = 0; jj < JB; ++jj) {
                                        const int c = 8 * (j0 + jj) + 2 * q4;
                                        svs[jj] = !kHR && want_sigma ? *reinterpret_cast<const float2*>(sw + cb + c) : make_float2(0.0f, 0.0f);
                                    }
#pragma unroll
                                    for (int jj = 0; jj < JB; ++jj) {
                                        const int j = j0 + jj;
                                        float a0 = acc[4 * j], a1 = acc[4 * j + 1], b0 = acc[4 * j + 2], b1 = acc[4 * j + 3];
                                        if (!kHR && relu) { a0 = fmaxf(a0, 0.0f); a1 = fmaxf(a1, 0.0f); b0 = fmaxf(b0, 0.0f); b1 = fmaxf(b1, 0.0f); }
                                        if (!kHR && want_sigma && cb + 8 * j < gm.n) {
                                            const float2 s = svs[jj];
                                            sacc_a = fmaf(a1, s.y, fmaf(a0, s.x, sacc_a));
                                            sacc_b = fmaf(b1, s.y, fmaf(b0, s.x, sacc_b));
                                        }
                                        uint32_t ha = pack_h2(a0, a1), hb = pack_h2(b0, b1);
                                        if constexpr (kHR) { ha = relu_h2(ha); hb = relu_h2(hb); }
                                        hreg[2 * j] = ha;
                                        hreg[2 * j + 1] = hb;
                                    }
                                }
                            };
                            if (relu && !want_sigma) epi(std::true_type{});
                            else epi(std::false_type{});
                            continue;
                        }
#pragma unroll
                        for (int j0 = 0; j0 < NM / 8; j0 += JB) {
                        float2 svs[JB];
#pragma unroll
                        for (int jj = 0; jj < JB; ++jj) {
                            const int c = 8 * (j0 + jj) + 2 * q4;
                            svs[jj] = want_sigma ? *reinterpret_cast<const float2*>(sw + cb + c) : make_float2(0.0f, 0.0f);
                        }
#pragma unroll
                        for (int jj = 0; jj < JB; ++jj) {
                            const int j = j0 + jj;
                            const bool in_n = cb + 8 * j < gm.n;
                            if (!in_n) continue;
                            float a0 = acc[4 * j], a1 = acc[4 * j + 1], b0 = acc[4 * j + 2], b1 = acc[4 * j + 3];
                            if (relu) { a0 = fmaxf(a0, 0.0f); a1 = fmaxf(a1, 0.0f); b0 = fmaxf(b0, 0.0f); b1 = fmaxf(b1, 0.0f); }
                            if (want_sigma && in_n) {
                                const float2 s = svs[jj];
                                sacc_a = fmaf(a1, s.y, fmaf(a0, s.x, sacc_a));
                                sacc_b = fmaf(b1, s.y, fmaf(b0, s.x, sacc_b));
                            }
                            const uint32_t ha = pack_h2(a0, a1), hb = pack_h2(b0, b1);
                            if (hold) { held[(2 * j) % (NM / 4)] = ha; held[(2 * j + 1) % (NM / 4)] = hb; }
                            else if (publish) put(cb + 8 * j + 2 * q4, ha, hb, a0, a1, b0, b1);
                        }
                        }
                        if (kWide && nch == 2 && ch == 1 && publish) {
#pragma unroll
                            for (int j = 0; j < NM / 8; ++j)
                                put(8 * j + 2 * q4, held[(2 * j) % (NM / 4)], held[(2 * j + 1) % (NM / 4)], 0.0f, 0.0f, 0.0f, 0.0f);
                        }
                    }
                    if (kMode == PP_DGRAD || rgb) return;
                    if (!kRegAct && publish) fence_proxy_async();    // generic-proxy stores to H -> visible to the tensor core
                    if (want_sigma) {
                        sacc_a += __shfl_xor_sync(0xffffffffu, sacc_a, 1);
                        sacc_a += __shfl_xor_sync(0xffffffffu, sacc_a, 2);
                        sacc_b += __shfl_xor_sync(0xffffffffu, sacc_b, 1);
                        sacc_b += __shfl_xor_sync(0xffffffffu, sacc_b, 2);
                        const float sbias = sw[L];                   // sigma bias is stored right after sigma_w
                        float sa = sacc_a + sbias, sb = sacc_b + sbias;
                        if (A.m.sigma_noise) {
                            if (row_a >= 0) sa = sa + A.m.sigma_noise[row_a];
                            if (row_b >= 0) sb = sb + A.m.sigma_noise[row_b];
                        }
                        sig_a = A.m.nd.softplus ? mn_softplus_shifted(sa) : fmaxf(sa, 0.0f);
                        sig_b = A.m.nd.softplus ? mn_softplus_shifted(sb) : fmaxf(sb, 0.0f);
                        if (q4 < 2) {
                            const int r = q4 ? rb : ra;
                            const int64_t row = q4 ? row_b : row_a, slot = q4 ? slot_b : slot_a;
                            const float s = q4 ? sb : sa, sg = q4 ? sig_b : sig_a;
                            if (kMode == PP_TRAIN_FWD) {
                                float* tf = A.tape_f32 + (size_t)tile * MN_TC_F32_ROWS * kTileM + r;
                                tf[MN_TC_F32_SIGMA * kTileM] = s;                           // pre-activation (with the density noise)
                                tf[MN_TC_F32_ID * kTileM] = (row >= 0 && A.m.nd.app > 0) ? A.m.src.index(row) : 0.0f;
                            }
                            if (A.m.sigma_only && row >= 0) {
                                const int64_t o = (A.m.scatter ? row : slot) * A.m.out_cols;
                                A.m.out[o] = A.m.slot_w ? sg * A.m.slot_w[slot] : sg;
                            }
                        }
                    }
                    if (!kRegAct) wg_sync();          // this layer's activations are complete before the next GEMM's MMAs read them
                };
                const int n = gm.n;
                if (n > 128) gemm(std::integral_constant<int, 256>{});
                else if (n > 64) gemm(std::integral_constant<int, 128>{});
                else if (n > 32) gemm(std::integral_constant<int, 64>{});
                else gemm(std::integral_constant<int, 32>{});
            }
        }
    }
    __syncthreads();
}
