// wgmma (sm_90a warpgroup MMA) wrappers: bf16 x bf16 -> fp32, M = 64 rows per warpgroup.
//
//   wgmma_ss<N, TA, TB>(d, a_desc, b_desc, scale_d)   A and B from shared memory (descriptors, see gmma_desc)
//   wgmma_rs<N, TB>(d, a_regs, b_desc, scale_d)       A from registers (the m64k16 fragment of the accumulator layout)
//
// TA / TB: 0 = K-major operand, 1 = MN-major operand.  scale_d == 0 overwrites d, != 0 accumulates into it.
// d holds N / 2 fp32 accumulators per thread: for n8 block j, d[4j], d[4j+1] are row (warp % 4) * 16 + lane / 4, columns
// 8j + 2 (lane % 4) + {0, 1}; d[4j+2], d[4j+3] the same columns of the row 8 further down.
#pragma once
#include <stdint.h>

// "+f" operands for d[i .. i+8k)
#define DOLO_F8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
#define DOLO_F16(i) DOLO_F8(i), DOLO_F8(i + 8)
#define DOLO_F32(i) DOLO_F16(i), DOLO_F16(i + 16)
#define DOLO_F64(i) DOLO_F32(i), DOLO_F32(i + 32)

namespace dolo {

template <int TA, int TB>
__device__ __forceinline__ void wgmma_ss_n16(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\twgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, %11, %12;\n\t}\n"
                 : DOLO_F8(0) : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_ss_n32(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\twgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, %20;\n\t}\n"
                 : DOLO_F16(0) : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_ss_n64(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\twgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n\t}\n"
                 : DOLO_F32(0) : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_ss_n128(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\twgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %68;\n\t}\n"
                 : DOLO_F64(0) : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
}
template <int TB>
__device__ __forceinline__ void wgmma_rs_n16(float* d, const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %13, 0;\n\twgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, p, 1, 1, %14;\n\t}\n"
                 : DOLO_F8(0) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d), "n"(TB));
}
template <int TB>
__device__ __forceinline__ void wgmma_rs_n32(float* d, const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\twgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1, %22;\n\t}\n"
                 : DOLO_F16(0) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d), "n"(TB));
}
template <int TB>
__device__ __forceinline__ void wgmma_rs_n64(float* d, const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\twgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, %38;\n\t}\n"
                 : DOLO_F32(0) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d), "n"(TB));
}

// N-generic entry points (N must be one of the instantiated widths)
template <int N, int TA, int TB>
__device__ __forceinline__ void wgmma_ss(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
    static_assert(N == 16 || N == 32 || N == 64 || N == 128, "wgmma_ss: unsupported N");
    if constexpr (N == 16) wgmma_ss_n16<TA, TB>(d, da, db, scale_d);
    else if constexpr (N == 32) wgmma_ss_n32<TA, TB>(d, da, db, scale_d);
    else if constexpr (N == 64) wgmma_ss_n64<TA, TB>(d, da, db, scale_d);
    else wgmma_ss_n128<TA, TB>(d, da, db, scale_d);
}
template <int N, int TB>
__device__ __forceinline__ void wgmma_rs(float* d, const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
    static_assert(N == 16 || N == 32 || N == 64, "wgmma_rs: unsupported N");
    if constexpr (N == 16) wgmma_rs_n16<TB>(d, a, db, scale_d);
    else if constexpr (N == 32) wgmma_rs_n32<TB>(d, a, db, scale_d);
    else wgmma_rs_n64<TB>(d, a, db, scale_d);
}

}  // namespace dolo
