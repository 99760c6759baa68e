// FP8 casts and the delayed-scaling recipe update (TransformerEngine's te.Linear input casts and DelayedScaling, used by
// fp8_autocast at pretrain.py:126-134 / finetune.py:90-98 of the reference).
//
//   cast:   q = satfinite_rne(fp32(x) * scale) to e4m3 (max 448) or e5m2 (max 57344), optionally also written transposed,
//           and max|x| folded into the slot's amax (atomicMax on the bit pattern: for non-negative floats the unsigned
//           order is the float order, and max is exact and independent of the order the blocks arrive in, so the
//           result is the same on every run).
//   update: per slot, amax = max(history) (NaN propagates, as torch.max); scale = fp8_max / amax when amax is finite and
//           > 0, else unchanged; scale_inv = 1 / scale; the history rolls by -1 and row 0 is zeroed.
#include <cuda_fp8.h>

#include "common.cuh"
#include "../../include/dolomite_b200.h"

namespace {

constexpr int CT = 64;  // tile edge of the cast (64 x 64 elements, 256 threads, 16 per thread)

template <int FMT, bool PLAIN, bool TRANS>
__global__ void __launch_bounds__(256) fp8_cast_kernel(const __nv_bfloat16* __restrict__ x, int64_t ldx, int64_t rows,
                                                       int64_t cols, const float* __restrict__ scale,
                                                       uint8_t* __restrict__ out, uint8_t* __restrict__ out_t,
                                                       float* __restrict__ amax) {
    __shared__ __align__(16) uint8_t tile[CT][CT + 16];
    __shared__ float wmax[8];
    const int64_t r0 = int64_t(blockIdx.y) * CT, c0 = int64_t(blockIdx.x) * CT;
    const int tr = threadIdx.x >> 2, tc = (threadIdx.x & 3) * 16;
    const int64_t r = r0 + tr, c = c0 + tc;
    const float s = __ldg(scale);
    float m = 0.f;
    uint4 q[1] = {make_uint4(0u, 0u, 0u, 0u)};
    if (r < rows && c < cols) {  // cols % 16 == 0: a 16-element chunk is wholly in range or wholly out
        const uint4* src = reinterpret_cast<const uint4*>(x + r * ldx + c);
        const uint4 v[2] = {__ldg(src), __ldg(src + 1)};
        const uint32_t* w = reinterpret_cast<const uint32_t*>(v);
        uint16_t* qh = reinterpret_cast<uint16_t*>(q);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const float a = dolo::bf16_lo(w[i]), b = dolo::bf16_hi(w[i]);
            m = fmaxf(m, fmaxf(fabsf(a), fabsf(b)));
            qh[i] = __nv_cvt_float2_to_fp8x2(make_float2(a * s, b * s), __NV_SATFINITE, FMT ? __NV_E5M2 : __NV_E4M3);
        }
        if (PLAIN) *reinterpret_cast<uint4*>(out + r * cols + c) = q[0];
    }
    if (TRANS) *reinterpret_cast<uint4*>(&tile[tr][tc]) = q[0];
    if (amax != nullptr) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        if ((threadIdx.x & 31) == 0) wmax[threadIdx.x >> 5] = m;
    }
    __syncthreads();
    if (amax != nullptr && threadIdx.x == 0) {
        float bm = wmax[0];
#pragma unroll
        for (int i = 1; i < 8; ++i) bm = fmaxf(bm, wmax[i]);
        if (bm > 0.f) atomicMax(reinterpret_cast<unsigned int*>(amax), __float_as_uint(bm));
    }
    if (TRANS) {
        // thread (tr, tc) writes column tr of the tile, rows tc .. tc + 15, as row c0 + tr of out_t [cols, rows]
        const int64_t orow = c0 + tr, ocol = r0 + tc;
        if (orow < cols && ocol < rows) {  // rows % 16 == 0
            uint4 t;
            uint8_t* tb = reinterpret_cast<uint8_t*>(&t);
#pragma unroll
            for (int i = 0; i < 16; ++i) tb[i] = tile[tc + i][tr];
            *reinterpret_cast<uint4*>(out_t + orow * rows + ocol) = t;
        }
    }
}

template <int FMT>
int launch_cast(const void* x, int64_t ldx, int64_t rows, int64_t cols, const float* scale, void* out, void* out_t,
                float* amax, cudaStream_t st) {
    const dim3 grid(unsigned((cols + CT - 1) / CT), unsigned((rows + CT - 1) / CT));
    const auto* xb = static_cast<const __nv_bfloat16*>(x);
    auto* o = static_cast<uint8_t*>(out);
    auto* ot = static_cast<uint8_t*>(out_t);
    if (out && out_t) fp8_cast_kernel<FMT, true, true><<<grid, 256, 0, st>>>(xb, ldx, rows, cols, scale, o, ot, amax);
    else if (out) fp8_cast_kernel<FMT, true, false><<<grid, 256, 0, st>>>(xb, ldx, rows, cols, scale, o, ot, amax);
    else fp8_cast_kernel<FMT, false, true><<<grid, 256, 0, st>>>(xb, ldx, rows, cols, scale, o, ot, amax);
    DOLO_LAUNCH_OK("fp8_cast");
    return DOLO_OK;
}

constexpr int MAX_HISTORY = 64;

__global__ void fp8_scaling_update_kernel(float* __restrict__ hist, int len, int64_t n, float* __restrict__ scale,
                                          float* __restrict__ scale_inv, float fp8_max) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float h[MAX_HISTORY];
    float amax = 0.f;
    for (int k = 0; k < len; ++k) {
        h[k] = hist[int64_t(k) * n + i];
        amax = (isnan(amax) || isnan(h[k])) ? __int_as_float(0x7fc00000) : fmaxf(amax, h[k]);
    }
    float s = scale[i];
    if (amax > 0.f && isfinite(amax)) s = __fdiv_rn(fp8_max, amax);
    scale[i] = s;
    scale_inv[i] = __fdiv_rn(1.f, s);
    // torch.roll(history, -1, 0), then row 0 = 0
    hist[i] = 0.f;
    for (int k = 1; k < len; ++k) hist[int64_t(k) * n + i] = h[(k + 1) % len];
}

}  // namespace

extern "C" int dolomite_b200_fp8_cast(const void* x, int64_t ldx, int64_t rows, int64_t cols, int fmt, const float* scale,
                                      void* out, void* out_t, float* amax, void* stream) {
    DOLO_REQUIRE(fmt == 0 || fmt == 1, "fp8_cast: format must be 0 (e4m3) or 1 (e5m2)");
    DOLO_REQUIRE(rows >= 0 && cols >= 0, "fp8_cast: negative dimension");
    DOLO_REQUIRE(out != nullptr || out_t != nullptr, "fp8_cast: no output");
    DOLO_REQUIRE(scale != nullptr, "fp8_cast: missing scale");
    DOLO_REQUIRE(cols % 16 == 0 && ldx % 8 == 0 && ldx >= cols, "fp8_cast: cols=%lld must be a multiple of 16 and ldx a "
                 "multiple of 8 >= cols", (long long)cols);
    DOLO_REQUIRE(out_t == nullptr || rows % 16 == 0, "fp8_cast: the transposed output needs rows %% 16 == 0 (rows=%lld)",
                 (long long)rows);
    const uintptr_t bits = reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(out_t);
    DOLO_REQUIRE((bits & 15) == 0 && (reinterpret_cast<uintptr_t>(amax) & 3) == 0, "fp8_cast: pointers must be 16-byte aligned");
    DOLO_REQUIRE((rows + CT - 1) / CT < 65536, "fp8_cast: too many rows");
    if (rows == 0 || cols == 0) return DOLO_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    return fmt ? launch_cast<1>(x, ldx, rows, cols, scale, out, out_t, amax, st)
               : launch_cast<0>(x, ldx, rows, cols, scale, out, out_t, amax, st);
}

extern "C" int dolomite_b200_fp8_scaling_update(float* amax_history, int history_len, int64_t n_slots, float* scale,
                                                float* scale_inv, float fp8_max, void* stream) {
    DOLO_REQUIRE(history_len >= 1 && history_len <= MAX_HISTORY, "fp8_scaling_update: history_len must be in [1, %d]",
                 MAX_HISTORY);
    DOLO_REQUIRE(n_slots >= 0, "fp8_scaling_update: negative slot count");
    DOLO_REQUIRE(fp8_max > 0.f, "fp8_scaling_update: fp8_max must be positive");
    if (n_slots == 0) return DOLO_OK;
    DOLO_REQUIRE(amax_history && scale && scale_inv, "fp8_scaling_update: null pointer");
    const int threads = 128;
    fp8_scaling_update_kernel<<<unsigned((n_slots + threads - 1) / threads), threads, 0, static_cast<cudaStream_t>(stream)>>>(
        amax_history, history_len, n_slots, scale, scale_inv, fp8_max);
    DOLO_LAUNCH_OK("fp8_scaling_update");
    return DOLO_OK;
}
