// HBM-bound kernels of the GPTDolomite training step: RMSNorm, RoPE, MLP activations, embedding, cross-entropy,
// bias-gradient column sums, residual adds and the flat-shard optimizer kernels.
// All are coalesced 16-byte vector kernels with warp-shuffle reductions; fp32 math, bf16 storage.
#include <type_traits>

#include "common.cuh"
#include "../../include/dolomite_b200.h"

using namespace dolo;

namespace {

constexpr int kThreads = 256;

__device__ __forceinline__ float block_sum(float v, float* red) {
    // red: >= 8 floats of shared memory.  Two barriers so `red` can be reused immediately.
    v = warp_sum(v);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (lane == 0) red[wid] = v;
    __syncthreads();
    float t = (lane < (blockDim.x >> 5)) ? red[lane] : 0.f;
    t = warp_sum(t);
    __syncthreads();
    return t;
}

// Deterministic column sums across the CTAs of a (1, CS, 1) cluster that split the rows of one column tile: every CTA
// leaves its per-column partials in shared memory, and rank 0 adds them in rank order (distributed shared memory) and
// applies the result to `out` -- the same order on every run, unlike one fp32 atomic per CTA.  Must be reached by every
// CTA of the cluster.
constexpr int kColsumCluster = 8;
__device__ __forceinline__ float ld_cluster_f32(const float* local_smem, uint32_t rank) {
    uint32_t remote;
    float v;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(local_smem)), "r"(rank));
    asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(remote) : "memory");
    return v;
}
__device__ __forceinline__ void cluster_colsum_apply(const float* part, float* out, bool ok, float scale) {
    cluster_sync_all();  // every CTA's partials are in its shared memory
    if (cluster_ctarank() == 0 && ok) {
        float s = 0.f;
        for (int r = 0; r < int(gridDim.y); ++r) s += ld_cluster_f32(part, uint32_t(r));
        *out += s * scale;
    }
    cluster_sync_all();  // the partials stay alive until rank 0 has read them
}
// Grid (column tiles, one cluster of row splits, segments): the row splits of segment z cover its rows in kColsumCluster
// equal parts (segment_rows); a dense launch is the one segment [0, T).
template <typename Kern, typename... Args>
static int launch_row_cluster(Kern kern, int col_tiles, int segments, cudaStream_t st, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(unsigned(col_tiles), kColsumCluster, unsigned(segments));
    cfg.blockDim = dim3(kThreads);
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 1;
    attr[0].val.clusterDim.y = kColsumCluster;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return int(cudaLaunchKernelEx(&cfg, kern, args...));
}

// Rows [r0, r1) of this CTA's row split.  seg == NULL: one segment [0, T) cut into rows_per_block rows per split.
// Otherwise segment blockIdx.z is rows [seg[z], seg[z + 1]) (an empty one gives every split an empty range).  Returns
// the offset of the segment's row of the per-segment sums, out_seg_stride floats apart (0 for the dense launch).
__device__ __forceinline__ int64_t segment_rows(const int* seg, int64_t T, int rows_per_block, int64_t out_seg_stride,
                                                int64_t& r0, int64_t& r1) {
    int64_t base = 0, n = T, rpb = rows_per_block, out_off = 0;
    if (seg != nullptr) {
        base = seg[blockIdx.z];
        n = seg[blockIdx.z + 1] - base;
        rpb = (n + kColsumCluster - 1) / kColsumCluster;
        out_off = int64_t(blockIdx.z) * out_seg_stride;
    }
    r0 = base + int64_t(blockIdx.y) * rpb;
    r1 = base + min(n, int64_t(blockIdx.y + 1) * rpb);
    return out_off;
}

__device__ __forceinline__ void unpack8(const uint4& v, float (&f)[8]) {
    f[0] = bf16_lo(v.x); f[1] = bf16_hi(v.x);
    f[2] = bf16_lo(v.y); f[3] = bf16_hi(v.y);
    f[4] = bf16_lo(v.z); f[5] = bf16_hi(v.z);
    f[6] = bf16_lo(v.w); f[7] = bf16_hi(v.w);
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
    uint4 v;
    v.x = pack_bf16(f[0], f[1]);
    v.y = pack_bf16(f[2], f[3]);
    v.z = pack_bf16(f[4], f[5]);
    v.w = pack_bf16(f[6], f[7]);
    return v;
}

// ------------------------------------------------------------------------------------------
// RMSNorm forward: one block per row (grid-stride), NV 16-byte vectors per thread held in registers.
// ------------------------------------------------------------------------------------------
template <int NV>
__global__ void __launch_bounds__(kThreads) rmsnorm_fwd_kernel(const uint4* __restrict__ x, const uint4* __restrict__ w,
                                                               uint4* __restrict__ y, float* __restrict__ rstd,
                                                               int64_t T, int H8, float eps, float inv_h) {
    __shared__ float red[8];
    for (int64_t row = blockIdx.x; row < T; row += gridDim.x) {
        const uint4* xr = x + row * H8;
        uint4 xv[NV];
        float ss = 0.f;
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const int idx = threadIdx.x + i * kThreads;
            if (idx < H8) {
                xv[i] = __ldg(xr + idx);
                float f[8];
                unpack8(xv[i], f);
#pragma unroll
                for (int j = 0; j < 8; ++j) ss += f[j] * f[j];
            }
        }
        ss = block_sum(ss, red);
        const float r = rsqrtf(ss * inv_h + eps);
        if (threadIdx.x == 0) rstd[row] = r;
        uint4* yr = y + row * H8;
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const int idx = threadIdx.x + i * kThreads;
            if (idx < H8) {
                float f[8], g[8];
                unpack8(xv[i], f);
                unpack8(__ldg(w + idx), g);
#pragma unroll
                for (int j = 0; j < 8; ++j) f[j] = g[j] * bf16_round(f[j] * r);  // weight * bf16(normalised)
                yr[idx] = pack8(f);
            }
        }
    }
}

// RMSNorm forward, one WARP per row (H <= 4096): lane l holds vectors l, l + 32, ... of the row in registers, all of them
// requested before the first use; the sum of squares is a warp reduction -- no shared memory, no block barrier.  The
// block-per-row kernel above keeps 8 CTAs x 5 KB = 40 KB of loads in flight per SM at H = 2560 (8 of its 32 registers hold
// data) and measured 4.6-4.9 TB/s; here 40 of ~64 registers hold data and 32 resident warps keep 160 KB in flight.
constexpr int kWarpRowThreads = 128;  // 4 rows per CTA, one CTA per 4 rows: no row loop, hence no imbalance between warps
template <int NVW>
__global__ void __launch_bounds__(kWarpRowThreads)
    rmsnorm_fwd_warp_kernel(const uint4* __restrict__ x, const uint4* __restrict__ w, uint4* __restrict__ y,
                            float* __restrict__ rstd, int64_t T, int H8, float eps, float inv_h) {
    const int lane = threadIdx.x & 31;
    const int64_t warp0 = int64_t(blockIdx.x) * (kWarpRowThreads / 32) + (threadIdx.x >> 5);
    const int64_t nwarps = int64_t(gridDim.x) * (kWarpRowThreads / 32);
    for (int64_t row = warp0; row < T; row += nwarps) {
        const uint4* xr = x + row * H8;
        uint4 xv[NVW];
#pragma unroll
        for (int i = 0; i < NVW; ++i) {
            const int idx = lane + i * 32;
            if (idx < H8) xv[i] = __ldg(xr + idx);
        }
        float ss = 0.f;
#pragma unroll
        for (int i = 0; i < NVW; ++i) {
            if (lane + i * 32 < H8) {
                float f[8];
                unpack8(xv[i], f);
#pragma unroll
                for (int j = 0; j < 8; ++j) ss += f[j] * f[j];
            }
        }
        ss = warp_sum(ss);
        const float r = rsqrtf(ss * inv_h + eps);
        if (lane == 0) rstd[row] = r;
        uint4* yr = y + row * H8;
#pragma unroll
        for (int i = 0; i < NVW; ++i) {
            const int idx = lane + i * 32;
            if (idx < H8) {
                float f[8], g[8];
                unpack8(xv[i], f);
                unpack8(__ldg(w + idx), g);
#pragma unroll
                for (int j = 0; j < 8; ++j) f[j] = g[j] * bf16_round(f[j] * r);  // weight * bf16(normalised)
                yr[idx] = pack8(f);
            }
        }
    }
}

// RMSNorm backward.  dx = r * (dy*w - xn * mean(dy*w*xn)),  dw += sum_rows dy * bf16(xn).
// Persistent blocks; per-thread dw partials in registers, written to workspace [gridDim.x, H].
template <int NV>
__global__ void __launch_bounds__(kThreads)
    rmsnorm_bwd_kernel(const uint4* __restrict__ dy, const uint4* __restrict__ x, const uint4* __restrict__ w,
                       const float* __restrict__ rstd, const uint4* __restrict__ dx_add, uint4* __restrict__ dx,
                       float* __restrict__ ws, int64_t T, int H8, float inv_h) {
    __shared__ float red[8];
    float dwacc[NV][8];
#pragma unroll
    for (int i = 0; i < NV; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) dwacc[i][j] = 0.f;

    for (int64_t row = blockIdx.x; row < T; row += gridDim.x) {
        const float r = rstd[row];
        uint4 xv[NV], gv[NV], av[NV];
        float dot = 0.f;
        // all three streams are requested before the block reduction, so only ONE global-memory latency per row is
        // exposed (the residual gradient used to be fetched after the reduction: 3.3 TB/s -> see profiles)
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const int idx = threadIdx.x + i * int(blockDim.x);
            if (idx < H8) {
                xv[i] = __ldg(x + row * H8 + idx);
                gv[i] = __ldg(dy + row * H8 + idx);
                if (dx_add != nullptr) av[i] = __ldg(dx_add + row * H8 + idx);
            }
        }
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const int idx = threadIdx.x + i * int(blockDim.x);
            if (idx < H8) {
                float xf[8], gf[8], wf[8];
                unpack8(xv[i], xf);
                unpack8(gv[i], gf);
                unpack8(__ldg(w + idx), wf);
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float xn = xf[j] * r;
                    dot += gf[j] * wf[j] * xn;
                    dwacc[i][j] += gf[j] * bf16_round(xn);
                }
            }
        }
        dot = block_sum(dot, red) * inv_h;
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const int idx = threadIdx.x + i * int(blockDim.x);
            if (idx < H8) {
                float xf[8], gf[8], wf[8], o[8];
                unpack8(xv[i], xf);
                unpack8(gv[i], gf);
                unpack8(__ldg(w + idx), wf);
#pragma unroll
                for (int j = 0; j < 8; ++j) o[j] = r * (gf[j] * wf[j] - xf[j] * r * dot);
                if (dx_add != nullptr) {
                    float a[8];
                    unpack8(av[i], a);
#pragma unroll
                    for (int j = 0; j < 8; ++j) o[j] += a[j];
                }
                dx[row * H8 + idx] = pack8(o);
            }
        }
    }
    float* wrow = ws + int64_t(blockIdx.x) * H8 * 8;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        const int idx = threadIdx.x + i * int(blockDim.x);
        if (idx < H8) {
            float4* p = reinterpret_cast<float4*>(wrow + idx * 8);
            p[0] = make_float4(dwacc[i][0], dwacc[i][1], dwacc[i][2], dwacc[i][3]);
            p[1] = make_float4(dwacc[i][4], dwacc[i][5], dwacc[i][6], dwacc[i][7]);
        }
    }
}

// out[c] += sum_p ws[p, c].  Block = 32 columns x 8 part-lanes (coalesced 128-byte rows, 8-way split of the sum).
__global__ void __launch_bounds__(256) reduce_partials_kernel(const float* __restrict__ ws, float* __restrict__ out,
                                                              int parts, int H, int ld) {
    __shared__ float sm[8][33];
    const int cx = threadIdx.x & 31, py = threadIdx.x >> 5;
    const int c = blockIdx.x * 32 + cx;
    float s = 0.f;
    if (c < H)
        for (int p = py; p < parts; p += 8) s += ws[int64_t(p) * ld + c];
    sm[py][cx] = s;
    __syncthreads();
    if (py == 0 && c < H) {
        float t = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) t += sm[i][cx];
        out[c] += t;
    }
}

// ------------------------------------------------------------------------------------------
// RoPE in place on packed qkv.  One block per token; each work item = one 8-wide vector of the first half of a
// rotated head slot and its partner in the second half.  bf16 rounding after every op like the eager reference.
// ------------------------------------------------------------------------------------------
// The block is sized to the work items of ONE token (launch: round_up(items, 32) threads), so the (group, slot, vector)
// decomposition -- integer divisions -- happens once per thread and the token loop only adds row strides.
template <typename PosT, int MAX_THREADS>  // 512: up to 128 registers (two tokens = 12 vectors in flight per thread); 1024: 64
__global__ void __launch_bounds__(MAX_THREADS)
    rope_kernel(__nv_bfloat16* __restrict__ qkv, int64_t row_stride, int64_t T, int n_groups, int q_per_group, int hd,
                const __nv_bfloat16* __restrict__ cos_t, const __nv_bfloat16* __restrict__ sin_t,
                const PosT* __restrict__ pos_ids, int64_t n_pos, float sin_sign) {
    const int half = hd >> 1;
    const int vec_per_half = half >> 3;
    const int rot_slots = q_per_group + 1;
    const int items = n_groups * rot_slots * vec_per_half;
    for (int it = threadIdx.x; it < items; it += blockDim.x) {
        const int v = it % vec_per_half;
        const int slot_lin = it / vec_per_half;
        const int g = slot_lin / rot_slots, sl = slot_lin % rot_slots;
        const int64_t slot_off = (int64_t(g) * (q_per_group + 2) + sl) * hd + v * 8;
        // two tokens per iteration: the position -> cos / sin -> arithmetic chain of one token is two dependent memory round
        // trips, so a second independent token doubles the bytes in flight per thread (the kernel sat at 0.61 of the copy peak)
        // y = x*cos + rotate_half(x)*sin with rotate_half(x) = cat(-x2, x1), every op rounded to bf16 like the eager reference
        // (position_embedding/rope.py:104-114 on bf16 tensors).  Native packed bf16 arithmetic (mul.bf16x2 / add.bf16x2): the
        // product of two bf16 values is exact in fp32, so the packed multiply rounds exactly once like `bf16(float(a) * float(b))`,
        // and a bf16 sum is exact in fp32 whenever it matters for the final rounding.  24 packed instructions per 16 outputs
        // instead of ~170 scalar ones: the fp32 version was issue-bound (0.60 of the copy bandwidth), not memory-bound.
        auto rotate = [&](int64_t t, uint4 a, uint4 b, uint4 ca, uint4 cb, uint4 sa, uint4 sb) {
            const __nv_bfloat162* x1 = reinterpret_cast<const __nv_bfloat162*>(&a);
            const __nv_bfloat162* x2 = reinterpret_cast<const __nv_bfloat162*>(&b);
            const __nv_bfloat162* c1 = reinterpret_cast<const __nv_bfloat162*>(&ca);
            const __nv_bfloat162* c2 = reinterpret_cast<const __nv_bfloat162*>(&cb);
            const __nv_bfloat162* s1 = reinterpret_cast<const __nv_bfloat162*>(&sa);
            const __nv_bfloat162* s2 = reinterpret_cast<const __nv_bfloat162*>(&sb);
            uint4 oa, ob;
            __nv_bfloat162* o1 = reinterpret_cast<__nv_bfloat162*>(&oa);
            __nv_bfloat162* o2 = reinterpret_cast<__nv_bfloat162*>(&ob);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                // backward: the transpose rotation dx1 = dy1*c1 + dy2*s2, dx2 = dy2*c2 - dy1*s1 (the halves of the sin
                // row trade places; the same thing for the reference's tables, whose halves are equal)
                const __nv_bfloat162 s1s = sin_sign < 0.f ? __hneg2(s2[j]) : s1[j];
                const __nv_bfloat162 s2s = sin_sign < 0.f ? __hneg2(s1[j]) : s2[j];
                o1[j] = __hadd2_rn(__hmul2_rn(x1[j], c1[j]), __hmul2_rn(__hneg2(x2[j]), s1s));  // _rn: never contracted into an fma
                o2[j] = __hadd2_rn(__hmul2_rn(x2[j], c2[j]), __hmul2_rn(x1[j], s2s));
            }
            __nv_bfloat16* base = qkv + t * row_stride + slot_off;
            *reinterpret_cast<uint4*>(base) = oa;
            *reinterpret_cast<uint4*>(base + half) = ob;
        };
        auto clamp_pos = [&](int64_t t) {
            int64_t pos = static_cast<int64_t>(__ldg(pos_ids + t));
            return pos < 0 ? int64_t(0) : (pos >= n_pos ? n_pos - 1 : pos);
        };
        const int64_t step = gridDim.x;
        int64_t t = blockIdx.x;
        for (; t + step < T; t += 2 * step) {
            const int64_t t1 = t + step;
            const int64_t p0 = clamp_pos(t), p1 = clamp_pos(t1);
            const __nv_bfloat16* b0 = qkv + t * row_stride + slot_off;
            const __nv_bfloat16* b1 = qkv + t1 * row_stride + slot_off;
            const uint4 a0 = *reinterpret_cast<const uint4*>(b0), h0 = *reinterpret_cast<const uint4*>(b0 + half);
            const uint4 a1 = *reinterpret_cast<const uint4*>(b1), h1 = *reinterpret_cast<const uint4*>(b1 + half);
            const uint4 ca0 = __ldg(reinterpret_cast<const uint4*>(cos_t + p0 * hd + v * 8));
            const uint4 cb0 = __ldg(reinterpret_cast<const uint4*>(cos_t + p0 * hd + half + v * 8));
            const uint4 sa0 = __ldg(reinterpret_cast<const uint4*>(sin_t + p0 * hd + v * 8));
            const uint4 sb0 = __ldg(reinterpret_cast<const uint4*>(sin_t + p0 * hd + half + v * 8));
            const uint4 ca1 = __ldg(reinterpret_cast<const uint4*>(cos_t + p1 * hd + v * 8));
            const uint4 cb1 = __ldg(reinterpret_cast<const uint4*>(cos_t + p1 * hd + half + v * 8));
            const uint4 sa1 = __ldg(reinterpret_cast<const uint4*>(sin_t + p1 * hd + v * 8));
            const uint4 sb1 = __ldg(reinterpret_cast<const uint4*>(sin_t + p1 * hd + half + v * 8));
            rotate(t, a0, h0, ca0, cb0, sa0, sb0);
            rotate(t1, a1, h1, ca1, cb1, sa1, sb1);
        }
        if (t < T) {
            const int64_t p0 = clamp_pos(t);
            const __nv_bfloat16* b0 = qkv + t * row_stride + slot_off;
            rotate(t, *reinterpret_cast<const uint4*>(b0), *reinterpret_cast<const uint4*>(b0 + half),
                   __ldg(reinterpret_cast<const uint4*>(cos_t + p0 * hd + v * 8)),
                   __ldg(reinterpret_cast<const uint4*>(cos_t + p0 * hd + half + v * 8)),
                   __ldg(reinterpret_cast<const uint4*>(sin_t + p0 * hd + v * 8)),
                   __ldg(reinterpret_cast<const uint4*>(sin_t + p0 * hd + half + v * 8)));
        }
    }
}

// ------------------------------------------------------------------------------------------
// MLP activations (hf_models/modeling_utils/activations/{base,glu}.py): one functor per function with its value f and
// its derivative d, used by one forward and one backward template in three forms (DOLO_ACT_PLAIN / _GLU /
// _SIGMOID_GLU, include/dolomite_b200.h).  fp32 math on bf16 storage.  Where torch's eager module rounds to bf16 more
// than once, f rounds at the same points (laplace, softsign, tanhshrink); d is the fp32 derivative with torch
// autograd's value at the non-differentiable points (bf16 inputs land on them often).
// ------------------------------------------------------------------------------------------
// MUFU ex2 + MUFU rcp (2 ulp fp32; the result is rounded to bf16 right after) instead of the ~10-instruction IEEE divide:
// the SwiGLU kernel is otherwise issue-bound next to its HBM time (168 M elements per layer).
__device__ __forceinline__ float sigmoidf_(float x) { return __fdividef(1.f, 1.f + __expf(-x)); }
__device__ __forceinline__ float tanh_fast(float z) {
    // tanh(z) = 1 - 2 / (1 + e^{2z}); MUFU ex2 + MUFU rcp, saturates cleanly for |z| large
    return 1.f - __fdividef(2.f, 1.f + __expf(2.f * z));
}

namespace act {
// min(max(x, lo), hi) that keeps a NaN (fminf / fmaxf return the other operand), as torch's clamp and relu do
__device__ __forceinline__ float clamp_nan(float x, float lo, float hi) { return x < lo ? lo : (x > hi ? hi : x); }
// elu / celu (alpha 1; CELU with alpha 1 is ELU) and selu: torch's elu kernel, x <= 0 ? expm1(x) * a * s : x * s
template <int kSelu>
struct EluT {
    static constexpr float s = kSelu ? 1.0507009873554804934193349852946f : 1.f;
    static constexpr float as = kSelu ? 1.0507009873554804934193349852946f * 1.6732632423543772848170429916717f : 1.f;
    __device__ static float f(float x) { return x <= 0.f ? expm1f(x) * as : x * s; }
    __device__ static float d(float x) { return x <= 0.f ? as * expf(x) : s; }
};
using Elu = EluT<0>;
using Selu = EluT<1>;
struct Gelu {  // exact erf
    __device__ static float f(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }
    __device__ static float d(float x) {
        return 0.5f * (1.f + erff(x * 0.70710678118654752f)) + x * 0.39894228040143268f * expf(-0.5f * x * x);
    }
};
// tanh-GELU (gelu_pytorch_tanh): y = 0.5 x (1 + tanh(k (x + c x^3))),  k = sqrt(2/pi), c = 0.044715
struct GeluTanh {
    __device__ static float f(float x) {
        const float z = 0.7978845608028654f * (x + 0.044715f * x * x * x);
        return 0.5f * x * (1.f + tanh_fast(z));
    }
    __device__ static float d(float x) {
        const float z = 0.7978845608028654f * (x + 0.044715f * x * x * x);
        const float t = tanh_fast(z);
        const float dz = 0.7978845608028654f * (1.f + 3.f * 0.044715f * x * x);
        return 0.5f * (1.f + t) + 0.5f * x * (1.f - t * t) * dz;
    }
};
struct HardShrink {  // lambda 0.5; zero on [-0.5, 0.5], ends included (value and gradient)
    __device__ static float f(float x) { return (x >= -0.5f && x <= 0.5f) ? 0.f : x; }
    __device__ static float d(float x) { return (x >= -0.5f && x <= 0.5f) ? 0.f : 1.f; }
};
struct HardSigmoid {
    __device__ static float f(float x) { return clamp_nan(x + 3.f, 0.f, 6.f) / 6.f; }
    __device__ static float d(float x) { return (x > -3.f && x < 3.f) ? 1.f / 6.f : 0.f; }
};
struct HardSwish {  // gradient x/3 + 1/2 inside (-3, 3); 0 at -3 and 1 at 3, as torch autograd gives
    __device__ static float f(float x) { return x * fminf(fmaxf(x + 3.f, 0.f), 6.f) / 6.f; }
    __device__ static float d(float x) { return x <= -3.f ? 0.f : (x < 3.f ? x / 3.f + 0.5f : 1.f); }
};
struct HardTanh {  // [-1, 1]; gradient 0 at the bounds
    __device__ static float f(float x) { return clamp_nan(x, -1.f, 1.f); }
    __device__ static float d(float x) { return (x > -1.f && x < 1.f) ? 1.f : 0.f; }
};
// transformers' LaplaceActivation, mu 0.707107, sigma 0.282095: 0.5 * (1 + erf((x - mu) / (sigma sqrt 2))), every eager
// op rounded to bf16 (the 0.5 * is exact).  torch's bf16 `x - mu` rounds the scalar mu to bf16 first (0.70703125): near
// erf = -1 the sum 1 + erf cancels, so that choice is visible in the result.
struct Laplace {
    static constexpr float mu = 0.70703125f;
    static constexpr float den = float(0.282095 * 1.4142135623730951);
    __device__ static float f(float x) {
        const float z = bf16_round(bf16_round(x - mu) / den);
        return 0.5f * bf16_round(1.f + bf16_round(erff(z)));
    }
    __device__ static float d(float x) {
        const float z = (x - 0.707107f) / den;
        return 0.56418958354775629f / den * expf(-z * z);  // 0.5 * 2/sqrt(pi) * exp(-z^2) / den
    }
};
struct LeakyRelu {  // slope 0.01; gradient 0.01 at 0
    __device__ static float f(float x) { return x > 0.f ? x : x * 0.01f; }
    __device__ static float d(float x) { return x > 0.f ? 1.f : 0.01f; }
};
struct LogSigmoid {
    __device__ static float f(float x) { return fminf(x, 0.f) - log1pf(expf(-fabsf(x))); }
    __device__ static float d(float x) {
        const float z = expf(-fabsf(x));
        return x < 0.f ? 1.f - z / (1.f + z) : z / (1.f + z);
    }
};
struct Mish {
    __device__ static float f(float x) { return x * tanhf(log1pf(expf(x))); }
    __device__ static float d(float x) {
        const float t = tanhf(log1pf(expf(x)));
        return t + x * (1.f / (1.f + expf(-x))) * (1.f - t * t);
    }
};
struct Relu {
    __device__ static float f(float x) { return x < 0.f ? 0.f : x; }
    __device__ static float d(float x) { return x > 0.f ? 1.f : 0.f; }
};
struct Relu2 {  // square(relu(x)): relu is exact, so one rounding
    __device__ static float f(float x) { const float r = x < 0.f ? 0.f : x; return r * r; }
    __device__ static float d(float x) { return x > 0.f ? 2.f * x : 0.f; }
};
struct Relu6 {  // hardtanh(0, 6): gradient 0 at both bounds
    __device__ static float f(float x) { return clamp_nan(x, 0.f, 6.f); }
    __device__ static float d(float x) { return (x > 0.f && x < 6.f) ? 1.f : 0.f; }
};
struct Sigmoid {
    __device__ static float f(float x) { return sigmoidf_(x); }
    __device__ static float d(float x) { const float s = sigmoidf_(x); return s * (1.f - s); }
};
struct Silu {
    __device__ static float f(float x) { return x * sigmoidf_(x); }
    __device__ static float d(float x) { const float s = sigmoidf_(x); return s * (1.f + x * (1.f - s)); }
};
struct Softplus {  // beta 1, threshold 20: linear (gradient 1) above the threshold
    __device__ static float f(float x) { return x > 20.f ? x : log1pf(expf(x)); }
    __device__ static float d(float x) { const float z = expf(x); return x > 20.f ? 1.f : z / (z + 1.f); }
};
struct SoftShrink {  // lambda 0.5; zero gradient on [-0.5, 0.5], ends included
    __device__ static float f(float x) { return (x >= -0.5f && x <= 0.5f) ? 0.f : (x > 0.f ? x - 0.5f : x + 0.5f); }
    __device__ static float d(float x) { return (x >= -0.5f && x <= 0.5f) ? 0.f : 1.f; }
};
struct SoftSign {  // x / (|x| + 1), the sum rounded first
    __device__ static float f(float x) { return x / bf16_round(fabsf(x) + 1.f); }
    __device__ static float d(float x) { const float a = 1.f + fabsf(x); return 1.f / (a * a); }
};
struct Tanh {
    __device__ static float f(float x) { return tanhf(x); }
    __device__ static float d(float x) { const float t = tanhf(x); return 1.f - t * t; }
};
struct TanhShrink {  // x - tanh(x), tanh rounded first
    __device__ static float f(float x) { return x - bf16_round(tanhf(x)); }
    __device__ static float d(float x) { const float t = tanhf(x); return t * t; }
};
}  // namespace act

// forward: plain y = f(x);  GLU x = [u | g], y = u * bf16(f(g));  sigmoid-GLU (torch's fused glu) y = u * f(g) rounded
// once.  Grid-stride over 16-byte vectors of y.
template <class Op, int Form>
__global__ void __launch_bounds__(kThreads) act_fwd_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, int64_t T,
                                                           int64_t F8) {
    const int64_t total = T * F8;
    for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += int64_t(gridDim.x) * blockDim.x) {
        float o[8];
        if constexpr (Form == DOLO_ACT_PLAIN) {
            unpack8(__ldg(x + i), o);
#pragma unroll
            for (int j = 0; j < 8; ++j) o[j] = Op::f(o[j]);
        } else {
            const int64_t t = i / F8, c = i - t * F8;
            float u[8], g[8];
            unpack8(__ldg(x + t * 2 * F8 + c), u);
            unpack8(__ldg(x + t * 2 * F8 + F8 + c), g);
#pragma unroll
            for (int j = 0; j < 8; ++j) o[j] = Form == DOLO_ACT_GLU ? u[j] * bf16_round(Op::f(g[j])) : u[j] * Op::f(g[j]);
        }
        y[i] = pack8(o);
    }
}

// dx of one row vector: plain dx = dy * f'(x);  GLU (both forms) du = dy * f(g), dg = dy * u * f'(g)
template <class Op, bool Glu>
__device__ __forceinline__ void act_bwd_vec(const uint4* __restrict__ dy, const uint4* __restrict__ x, int64_t t,
                                            int64_t c, int64_t F8, float (&o)[Glu ? 2 : 1][8]) {
    float d[8];
    unpack8(__ldg(dy + t * F8 + c), d);
    if constexpr (Glu) {
        float u[8], g[8];
        unpack8(__ldg(x + t * 2 * F8 + c), u);
        unpack8(__ldg(x + t * 2 * F8 + F8 + c), g);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            o[0][j] = d[j] * Op::f(g[j]);
            o[1][j] = d[j] * u[j] * Op::d(g[j]);
        }
    } else {
        float xf[8];
        unpack8(__ldg(x + t * F8 + c), xf);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[0][j] = d[j] * Op::d(xf[j]);
    }
}

template <class Op, bool Glu>
__global__ void __launch_bounds__(kThreads) act_bwd_kernel(const uint4* __restrict__ dy, const uint4* __restrict__ x,
                                                           uint4* __restrict__ dx, int64_t T, int64_t F8) {
    constexpr int NP = Glu ? 2 : 1;
    const int64_t total = T * F8;
    for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += int64_t(gridDim.x) * blockDim.x) {
        const int64_t t = i / F8, c = i - t * F8;
        float o[NP][8];
        act_bwd_vec<Op, Glu>(dy, x, t, c, F8, o);
#pragma unroll
        for (int p = 0; p < NP; ++p) dx[t * NP * F8 + p * F8 + c] = pack8(o[p]);
    }
}

// Backward that also accumulates the bias gradient of the producing linear layer (column sums of the bf16 dx it
// writes): saves the separate pass that re-read the whole dx.  Block = 32 column vectors (256 columns of each half)
// x 8 row lanes over `rows_per_block` rows; per-thread fp32 column sums, smem combine, and the row splits of a column
// tile (one cluster) combined in a fixed order (cluster_colsum_apply).  With a segment table (grouped MoE rows) the
// grid's z enumerates the segments and each gets its own bias-gradient row (segment_rows).
template <class Op, bool Glu>
__global__ void __launch_bounds__(kThreads)
    act_bwd_bias_kernel(const uint4* __restrict__ dy, const uint4* __restrict__ x, uint4* __restrict__ dx,
                        float* __restrict__ dbias, int64_t T, int64_t F8, int rows_per_block,
                        const int* __restrict__ seg, int64_t dbias_seg_stride) {
    constexpr int NP = Glu ? 2 : 1;
    __shared__ float sm[8][NP][256];
    const int lane = threadIdx.x & 31, rl = threadIdx.x >> 5;
    const int64_t c = int64_t(blockIdx.x) * 32 + lane;
    int64_t r0, r1;
    float* const dbias_seg = dbias + segment_rows(seg, T, rows_per_block, dbias_seg_stride, r0, r1);
    float s[NP][8];
#pragma unroll
    for (int p = 0; p < NP; ++p)
#pragma unroll
        for (int j = 0; j < 8; ++j) s[p][j] = 0.f;
    if (c < F8) {
        for (int64_t t = r0 + rl; t < r1; t += 8) {
            float o[NP][8];
            act_bwd_vec<Op, Glu>(dy, x, t, c, F8, o);
#pragma unroll
            for (int p = 0; p < NP; ++p) {
                const uint4 pk = pack8(o[p]);
                dx[t * NP * F8 + p * F8 + c] = pk;
                unpack8(pk, o[p]);  // the bias gradient sums the bf16 values autograd would see
#pragma unroll
                for (int j = 0; j < 8; ++j) s[p][j] += o[p][j];
            }
        }
    }
#pragma unroll
    for (int p = 0; p < NP; ++p)
#pragma unroll
        for (int j = 0; j < 8; ++j) sm[rl][p][lane * 8 + j] = s[p][j];
    __syncthreads();
    __shared__ float part[NP][256];
    const int col = threadIdx.x;
#pragma unroll
    for (int p = 0; p < NP; ++p) {
        float a = 0.f;
#pragma unroll
        for (int w = 0; w < 8; ++w) a += sm[w][p][col];
        part[p][col] = a;
    }
    const int64_t gc = int64_t(blockIdx.x) * 256 + col;
    const bool ok = gc < F8 * 8;
#pragma unroll
    for (int p = 0; p < NP; ++p) cluster_colsum_apply(&part[p][col], dbias_seg + (ok ? p * F8 * 8 + gc : 0), ok, 1.f);
}

// ------------------------------------------------------------------------------------------
// LayerNorm (normalization_function layernorm = torch.nn.LayerNorm): fp32 statistics, ONE rounding to bf16 at the end
//   y = bf16( (x - mean) * rstd * w + b )
// Same block-per-row structure as the RMSNorm kernels; mean and rstd are saved for backward.
// ------------------------------------------------------------------------------------------
template <int NV>
__global__ void __launch_bounds__(kThreads)
    layernorm_fwd_kernel(const uint4* __restrict__ x, const uint4* __restrict__ w, const uint4* __restrict__ b,
                         uint4* __restrict__ y, float* __restrict__ mean, float* __restrict__ rstd, int64_t T, int H8,
                         float eps, float inv_h) {
    __shared__ float red[8];
    for (int64_t row = blockIdx.x; row < T; row += gridDim.x) {
        uint4 xv[NV];
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const int idx = threadIdx.x + i * kThreads;
            if (idx < H8) {
                xv[i] = __ldg(x + row * H8 + idx);
                float f[8];
                unpack8(xv[i], f);
#pragma unroll
                for (int j = 0; j < 8; ++j) s += f[j];
            }
        }
        const float mu = block_sum(s, red) * inv_h;
        float ss = 0.f;
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const int idx = threadIdx.x + i * kThreads;
            if (idx < H8) {
                float f[8];
                unpack8(xv[i], f);
#pragma unroll
                for (int j = 0; j < 8; ++j) ss += (f[j] - mu) * (f[j] - mu);
            }
        }
        const float r = rsqrtf(block_sum(ss, red) * inv_h + eps);
        if (threadIdx.x == 0) {
            mean[row] = mu;
            rstd[row] = r;
        }
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const int idx = threadIdx.x + i * kThreads;
            if (idx < H8) {
                float f[8], g[8], bb[8];
                unpack8(xv[i], f);
                unpack8(__ldg(w + idx), g);
#pragma unroll
                for (int j = 0; j < 8; ++j) f[j] = (f[j] - mu) * r * g[j];
                if (b != nullptr) {
                    unpack8(__ldg(b + idx), bb);
#pragma unroll
                    for (int j = 0; j < 8; ++j) f[j] += bb[j];
                }
                y[row * H8 + idx] = pack8(f);
            }
        }
    }
}

// dx = rstd * (g*w - mean(g*w) - xhat * mean(g*w*xhat)) [+ dx_add];  dw += sum_rows g*xhat;  db += sum_rows g.
// Per-thread dw / db partials go to the workspace [gridDim.x][2][H] (reduced by reduce_partials_kernel).
template <int NV>
__global__ void __launch_bounds__(kThreads)
    layernorm_bwd_kernel(const uint4* __restrict__ dy, const uint4* __restrict__ x, const uint4* __restrict__ w,
                         const float* __restrict__ mean, const float* __restrict__ rstd, const uint4* __restrict__ dx_add,
                         uint4* __restrict__ dx, float* __restrict__ ws, int64_t T, int H8, float inv_h) {
    __shared__ float red[8];
    float dwacc[NV][8], dbacc[NV][8];
#pragma unroll
    for (int i = 0; i < NV; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) dwacc[i][j] = dbacc[i][j] = 0.f;
    for (int64_t row = blockIdx.x; row < T; row += gridDim.x) {
        const float mu = mean[row], r = rstd[row];
        uint4 xv[NV], gv[NV];
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const int idx = threadIdx.x + i * kThreads;
            if (idx < H8) {
                xv[i] = __ldg(x + row * H8 + idx);
                gv[i] = __ldg(dy + row * H8 + idx);
                float xf[8], gf[8], wf[8];
                unpack8(xv[i], xf);
                unpack8(gv[i], gf);
                unpack8(__ldg(w + idx), wf);
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float xh = (xf[j] - mu) * r;
                    const float gw = gf[j] * wf[j];
                    s1 += gw;
                    s2 += gw * xh;
                    dwacc[i][j] += gf[j] * xh;
                    dbacc[i][j] += gf[j];
                }
            }
        }
        s1 = block_sum(s1, red) * inv_h;
        s2 = block_sum(s2, red) * inv_h;
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const int idx = threadIdx.x + i * kThreads;
            if (idx < H8) {
                float xf[8], gf[8], wf[8], o[8];
                unpack8(xv[i], xf);
                unpack8(gv[i], gf);
                unpack8(__ldg(w + idx), wf);
#pragma unroll
                for (int j = 0; j < 8; ++j) o[j] = r * (gf[j] * wf[j] - s1 - (xf[j] - mu) * r * s2);
                if (dx_add != nullptr) {
                    float a[8];
                    unpack8(__ldg(dx_add + row * H8 + idx), a);
#pragma unroll
                    for (int j = 0; j < 8; ++j) o[j] += a[j];
                }
                dx[row * H8 + idx] = pack8(o);
            }
        }
    }
    float* wrow = ws + int64_t(blockIdx.x) * 2 * H8 * 8;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        const int idx = threadIdx.x + i * kThreads;
        if (idx < H8) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                wrow[idx * 8 + j] = dwacc[i][j];
                wrow[H8 * 8 + idx * 8 + j] = dbacc[i][j];
            }
        }
    }
}

// ------------------------------------------------------------------------------------------
// Embedding
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
    embedding_fwd_kernel(const int64_t* __restrict__ ids, const uint4* __restrict__ wte, uint4* __restrict__ out,
                         int64_t T, int H8, int64_t V, float scale, int apply_scale) {
    for (int64_t t = blockIdx.x; t < T; t += gridDim.x) {
        int64_t id = ids[t];
        id = id < 0 ? 0 : (id >= V ? V - 1 : id);
        const uint4* src = wte + id * H8;
        for (int i = threadIdx.x; i < H8; i += blockDim.x) {
            uint4 v = __ldg(src + i);
            if (apply_scale) {
                float f[8];
                unpack8(v, f);
#pragma unroll
                for (int j = 0; j < 8; ++j) f[j] *= scale;
                v = pack8(f);
            }
            out[t * H8 + i] = v;
        }
    }
}

// wte(ids) + NEFTune noise (model_wrapper/base.py:246-267 in training mode): x + zeros_like(x).uniform_(-mag, mag) on a bf16
// x, with the rounding points of torch's CUDA uniform kernel (ATen/native/cuda/DistributionTemplates.h `uniform_kernel`):
//   from = bf16(-mag), to = bf16(mag), range = fp32(bf16(to - from)),
//   v = bf16(u * range + from) in fp32 with u in (0, 1] -- here __fmul_rn then __fadd_rn: no contraction to an FMA --
//   v == to -> from, out = bf16(x + v).
// u = ((h >> 8) + 1) * 2^-24 with h = dropout_hash_flat(t * H + c, key0, key1): 2^24 equally likely values in (0, 1], each
// exact in fp32.  The caller passes bf16(-mag) / bf16(mag) / range as floats (`from`, `to`, `range`).
__global__ void __launch_bounds__(kThreads)
    embedding_fwd_neft_kernel(const int64_t* __restrict__ ids, const uint4* __restrict__ wte, uint4* __restrict__ out,
                              int64_t T, int H8, int64_t V, uint32_t key0, uint32_t key1, float from, float to, float range) {
    for (int64_t t = blockIdx.x; t < T; t += gridDim.x) {
        int64_t id = ids[t];
        id = id < 0 ? 0 : (id >= V ? V - 1 : id);
        const uint4* src = wte + id * H8;
        for (int i = threadIdx.x; i < H8; i += blockDim.x) {
            float f[8];
            unpack8(__ldg(src + i), f);
            const uint64_t e0 = (uint64_t(t) * uint64_t(H8) + uint64_t(i)) * 8;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const uint32_t h = dropout_hash_flat(e0 + j, key0, key1);
                const float u = float((h >> 8) + 1u) * 5.9604644775390625e-8f;  // 2^-24
                float v = bf16_round(__fadd_rn(__fmul_rn(u, range), from));
                v = v == to ? from : v;
                f[j] = __fadd_rn(f[j], v);
            }
            out[t * H8 + i] = pack8(f);
        }
    }
}

// One warp per token.  The warp of the FIRST token with a given id owns that row of dwte and adds the rows of all tokens
// with that id in ascending token order: a fixed summation order (bit-identical runs) without atomics.
__device__ __forceinline__ int64_t clamp_id(int64_t id, int64_t V) { return id < 0 ? 0 : (id >= V ? V - 1 : id); }
__global__ void __launch_bounds__(kThreads)
    embedding_bwd_kernel(const int64_t* __restrict__ ids, const uint4* __restrict__ dout, float* __restrict__ dwte,
                         int64_t T, int H8, int64_t V, float scale) {
    const int lane = threadIdx.x & 31;
    const int64_t t = int64_t(blockIdx.x) * (kThreads / 32) + (threadIdx.x >> 5);
    if (t >= T) return;  // uniform per warp
    const int64_t id = clamp_id(ids[t], V);
    for (int64_t base = 0; base < t; base += 32) {
        const int64_t u = base + lane;
        if (__any_sync(0xffffffffu, u < t && clamp_id(ids[u], V) == id)) return;  // an earlier token owns the row
    }
    float4* dst = reinterpret_cast<float4*>(dwte + id * H8 * 8);
    for (int64_t base = t; base < T; base += 32) {
        const int64_t u0 = base + lane;
        uint32_t m = __ballot_sync(0xffffffffu, u0 < T && clamp_id(ids[u0], V) == id);
        while (m) {
            const int64_t u = base + (__ffs(m) - 1);
            m &= m - 1;
            for (int i = lane; i < H8; i += 32) {
                float f[8];
                unpack8(__ldg(dout + u * H8 + i), f);
                float4 a = dst[2 * i], b = dst[2 * i + 1];
                a.x += f[0] * scale; a.y += f[1] * scale; a.z += f[2] * scale; a.w += f[3] * scale;
                b.x += f[4] * scale; b.y += f[5] * scale; b.z += f[6] * scale; b.w += f[7] * scale;
                dst[2 * i] = a;
                dst[2 * i + 1] = b;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------
// Cross entropy: one block (or cluster) per row, row held in registers between the reduction and the gradient write.
// ------------------------------------------------------------------------------------------
constexpr int kCeThreads = 256;  // two CTAs per SM: one loads / stores its row while the other is in its reduction phases

__global__ void ce_count_kernel(const int64_t* __restrict__ labels, int64_t T, int64_t ignore_index,
                                float* __restrict__ scratch) {
    // single block; scratch[0] = n_valid, scratch[1] = 0 (loss accumulator)
    __shared__ float red[32];
    float c = 0.f;
    for (int64_t i = threadIdx.x; i < T; i += blockDim.x) c += (labels[i] != ignore_index) ? 1.f : 0.f;
    c = warp_sum(c);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x < 32) {
        float t = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
        t = warp_sum(t);
        if (threadIdx.x == 0) {
            scratch[0] = t;
            scratch[1] = 0.f;
        }
    }
}

// Row-resident cross entropy: a row (or, for wide vocabularies, 1/SPLIT of a row per CTA of a SPLIT-CTA cluster) is read
// from HBM ONCE into registers (NV 16-byte vectors per thread), max and sum-of-exponentials are reduced in the block (and
// across the cluster through distributed shared memory), and the gradient row is written from the same registers: 4 B per
// logit of traffic, the algorithmic minimum.  logits and dlogits may alias, hence no __restrict__ / __ldg on them.
__device__ __forceinline__ float ce_block_reduce(float v, float* red, bool is_max) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    v = is_max ? warp_max(v) : warp_sum(v);
    if (lane == 0) red[wid] = v;
    __syncthreads();
    float t = lane < (kCeThreads / 32) ? red[lane] : (is_max ? -INFINITY : 0.f);
    t = is_max ? warp_max(t) : warp_sum(t);
    __syncthreads();
    return t;
}
__device__ __forceinline__ void st_cluster_f32(float* local_smem, uint32_t rank, float v) {
    uint32_t remote;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(local_smem)), "r"(rank));
    asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(remote), "f"(v) : "memory");
}

// TAIL: V % 8 != 0.  The row's last vector (index V8 - 1) then holds only V - 8 (V8 - 1) logits; its other lanes are
// left out of the max and the sum and get a zero gradient.  Without TAIL the kernel is the plain full-vector one.
template <int NV, int SPLIT, bool TAIL>
__global__ void __launch_bounds__(kCeThreads, 2)
    ce_rows_kernel(const uint4* logits, int64_t ld8, const int64_t* __restrict__ labels, uint4* dlogits,
                   float* __restrict__ loss_tok, const float* __restrict__ scratch, int64_t T, int64_t V,
                   int64_t ignore_index, float logit_scale, float grad_scale) {
    __shared__ float red[kCeThreads / 32];
    __shared__ float xch[2][4];  // [max | sum][cluster rank]: written by every CTA of the cluster (DSMEM)
    const int crank = SPLIT > 1 ? int(cluster_ctarank()) : 0;
    const int64_t V8 = (V + 7) >> 3;
    const int64_t vlast = V8 - 1;
    const int tail = int(V - 8 * vlast);  // valid lanes of the last vector, 1 .. 8
    const int64_t per = (V8 + SPLIT - 1) / SPLIT;
    const int64_t v_lo = crank * per, v_hi = min(V8, v_lo + per);
    const float n_valid = scratch[0];
    const float gs = n_valid > 0.f ? grad_scale / n_valid : 0.f;
    const int64_t n_clusters = gridDim.x / SPLIT;
    for (int64_t row = blockIdx.x / SPLIT; row < T; row += n_clusters) {
        const uint4* lr = logits + row * ld8;
        uint4* dr = dlogits + row * ld8;
        const int64_t label = labels[row];
        if (label == ignore_index) {  // uniform per cluster: zero gradient row
            for (int64_t i = v_lo + threadIdx.x; i < v_hi; i += kCeThreads) dr[i] = make_uint4(0, 0, 0, 0);
            if (crank == 0 && threadIdx.x == 0) loss_tok[row] = 0.f;
            continue;
        }
        if (label < 0 || label >= V) {  // torch's cross_entropy asserts on the device for this as well
            if (threadIdx.x == 0 && crank == 0)
                printf("[dolomite_b200] cross_entropy: label %lld of row %lld is outside [0, %lld)\n", (long long)label,
                       (long long)row, (long long)V);
            __trap();
        }
        uint4 v[NV];
#pragma unroll
        for (int k = 0; k < NV; ++k) {
            const int64_t i = v_lo + k * kCeThreads + threadIdx.x;
            if (i < v_hi) v[k] = lr[i];
        }
        // everything in log2 units: x2 = x * (logit_scale * log2 e), so that exp() is ONE ex2.approx after one FFMA
        const float scale2 = logit_scale * 1.4426950408889634f;
        float m = -INFINITY;
#pragma unroll
        for (int k = 0; k < NV; ++k) {
            const int64_t i = v_lo + k * kCeThreads + threadIdx.x;
            if (i < v_hi) {
                float f[8];
                unpack8(v[k], f);
                const int nl = TAIL && i == vlast ? tail : 8;
#pragma unroll
                for (int j = 0; j < 8; ++j) m = fmaxf(m, !TAIL || j < nl ? f[j] * scale2 : -INFINITY);
            }
        }
        m = ce_block_reduce(m, red, true);
        if (SPLIT > 1) {
            if (threadIdx.x < SPLIT) st_cluster_f32(&xch[0][crank], threadIdx.x, m);
            cluster_sync_all();
#pragma unroll
            for (int c = 0; c < SPLIT; ++c) m = fmaxf(m, xch[0][c]);
        }
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < NV; ++k) {
            const int64_t i = v_lo + k * kCeThreads + threadIdx.x;
            if (i < v_hi) {
                float f[8];
                unpack8(v[k], f);
                const int nl = TAIL && i == vlast ? tail : 8;
#pragma unroll
                for (int j = 0; j < 8; ++j)
                    if (!TAIL || j < nl) s += fast_exp2(fmaf(f[j], scale2, -m));
            }
        }
        s = ce_block_reduce(s, red, false);
        if (SPLIT > 1) {
            if (threadIdx.x < SPLIT) st_cluster_f32(&xch[1][crank], threadIdx.x, s);
            cluster_sync_all();
            s = 0.f;
#pragma unroll
            for (int c = 0; c < SPLIT; ++c) s += xch[1][c];
        }
        const float lse2 = m + __log2f(s);  // log2 units
        const float gmul = gs * logit_scale;
        const int64_t lvec = label >> 3;
        const int lsub = int(label & 7);
#pragma unroll
        for (int k = 0; k < NV; ++k) {
            const int64_t i = v_lo + k * kCeThreads + threadIdx.x;
            if (i < v_hi) {
                float f[8];
                unpack8(v[k], f);
                // (compile-time indices only: a run-time index into f[] would move the array to local memory -- the ncu
                //  capture of the first version showed two STL.128 + LDL per vector and long-scoreboard stalls on them)
                const bool has_label = (i == lvec);
                if (has_label) {
                    float xl = 0.f;
#pragma unroll
                    for (int j = 0; j < 8; ++j) xl = (j == lsub) ? f[j] : xl;
                    loss_tok[row] = (lse2 - xl * scale2) * 0.6931471805599453f;
                }
                const int nl = TAIL && i == vlast ? tail : 8;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float pj = fast_exp2(fmaf(f[j], scale2, -lse2));
                    f[j] = ((has_label && j == lsub) ? pj - 1.f : pj) * gmul;
                    if (TAIL && j >= nl) f[j] = 0.f;
                }
                dr[i] = pack8(f);
            }
        }
        // no third cluster barrier: xch[0] of this row was read before barrier 2 and is rewritten only after it; xch[1] was
        // read before the next row's barrier 1 and is rewritten only after it
    }
}

template <int NV, int SPLIT, bool TAIL>
int launch_ce_rows(const void* logits, int64_t ldl, const int64_t* labels, void* dlogits, float* loss_tok,
                   const float* scratch, int64_t T, int64_t V, int64_t ignore_index, float logit_scale, float grad_scale,
                   cudaStream_t st) {
    auto kern = ce_rows_kernel<NV, SPLIT, TAIL>;
    int64_t clusters = 2 * int64_t(dolo_num_sms()) / SPLIT;  // two 256-thread CTAs per SM (a row lives in a CTA's registers)
    if (clusters > T) clusters = T;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(unsigned(clusters * SPLIT));
    cfg.blockDim = dim3(kCeThreads);
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = SPLIT;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = SPLIT > 1 ? 1 : 0;
    DOLO_CUDA_OK(cudaLaunchKernelEx(&cfg, kern, static_cast<const uint4*>(logits), ldl / 8, labels,
                                    static_cast<uint4*>(dlogits), loss_tok, scratch, T, V, ignore_index, logit_scale,
                                    grad_scale));
    return DOLO_OK;
}

__global__ void ce_mean_kernel(const float* __restrict__ loss_tok, int64_t T, const float* __restrict__ scratch,
                               float* __restrict__ loss_mean) {
    // single block, deterministic order
    __shared__ float red[32];
    float s = 0.f;
    for (int64_t i = threadIdx.x; i < T; i += blockDim.x) s += loss_tok[i];
    s = warp_sum(s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x < 32) {
        float t = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
        t = warp_sum(t);
        if (threadIdx.x == 0) loss_mean[0] = scratch[0] > 0.f ? t / scratch[0] : 0.f;
    }
}

// ------------------------------------------------------------------------------------------
// column sums: grid (col tiles of 256 columns, row splits = one cluster).  each thread owns 8 columns (one 16-B vector)
// of 32 lanes; 8 warps stride rows; smem combine; row splits combined in a fixed order (cluster_colsum_apply).  With a
// segment table, grid z enumerates the segments (segment_rows): per-expert bias gradients of grouped MoE rows.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
    colsum_kernel(const __nv_bfloat16* __restrict__ x, int64_t ldx, float* __restrict__ out, int64_t T, int64_t N,
                  int rows_per_block, float scale, const int* __restrict__ seg, int64_t out_seg_stride) {
    __shared__ float sm[8][256];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int64_t col = int64_t(blockIdx.x) * 256 + lane * 8;
    int64_t r0, r1;
    float* const out_seg = out + segment_rows(seg, T, rows_per_block, out_seg_stride, r0, r1);
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    if (col < N) {
        for (int64_t r = r0 + wid; r < r1; r += 8) {
            float f[8];
            unpack8(__ldg(reinterpret_cast<const uint4*>(x + r * ldx + col)), f);
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[j] += f[j];
        }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) sm[wid][lane * 8 + j] = acc[j];
    __syncthreads();
    __shared__ float part[256];
    const int c = threadIdx.x;
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += sm[w][c];
    part[c] = s;
    const int64_t gc = int64_t(blockIdx.x) * 256 + c;
    const bool ok = gc < N;
    cluster_colsum_apply(&part[c], out_seg + (ok ? gc : 0), ok, scale);
}

__global__ void __launch_bounds__(kThreads) add_scaled_kernel(const uint4* __restrict__ a, const uint4* __restrict__ b,
                                                              uint4* __restrict__ out, float alpha, int64_t n8) {
    for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n8; i += int64_t(gridDim.x) * blockDim.x) {
        float x[8], y[8];
        unpack8(a[i], x);
        unpack8(b[i], y);
#pragma unroll
        for (int j = 0; j < 8; ++j) x[j] = x[j] + bf16_round(alpha * y[j]);
        out[i] = pack8(x);
    }
}

// ------------------------------------------------------------------------------------------
// optimizer kernels on flat fp32 shards
// ------------------------------------------------------------------------------------------
// sum of squares in two launches with a fixed reduction tree: kSumsqBlocks grid-stride partials (fixed grid, so every
// element always lands in the same partial), then one block adds them in a fixed order -- bit-identical runs.
constexpr int kSumsqBlocks = 1024;
__global__ void __launch_bounds__(kThreads)
    sumsq_partial_kernel(const float* __restrict__ g, int64_t n, float* __restrict__ partials) {
    __shared__ float red[8];
    float s = 0.f;
    const int64_t n4 = n >> 2;
    const float4* g4 = reinterpret_cast<const float4*>(g);
    for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n4; i += int64_t(gridDim.x) * blockDim.x) {
        const float4 v = __ldg(g4 + i);
        s += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
    }
    for (int64_t i = (n4 << 2) + int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
         i += int64_t(gridDim.x) * blockDim.x)
        s += g[i] * g[i];
    s = block_sum(s, red);
    if (threadIdx.x == 0) partials[blockIdx.x] = s;
}
__global__ void __launch_bounds__(kThreads) sumsq_final_kernel(const float* __restrict__ partials, float* __restrict__ out) {
    __shared__ float red[8];
    float s = 0.f;
    for (int i = threadIdx.x; i < kSumsqBlocks; i += kThreads) s += partials[i];
    s = block_sum(s, red);
    if (threadIdx.x == 0) out[0] += s;
}

__global__ void clip_coef_kernel(const float* sumsq, float max_norm, float* coef, float* norm_out) {
    const float norm = sqrtf(sumsq[0]);
    if (norm_out) norm_out[0] = norm;
    float c = 1.f;
    if (max_norm > 0.f) {
        // torch.clamp(max_norm / (norm + 1e-6), max=1): a NaN norm gives a NaN coefficient (fminf would give 1), so a NaN
        // gradient poisons every parameter as it does in the reference instead of updating the finite ones unclipped
        const float r = max_norm / (norm + 1e-6f);
        c = r >= 1.f ? 1.f : r;
    }
    coef[0] = c;
}

__global__ void __launch_bounds__(kThreads)
    adamw_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                 __nv_bfloat16* __restrict__ pb, int64_t n, float lr, float b1, float b2, float eps, float wd,
                 float bc1, float bc2_sqrt, const float* __restrict__ clip) {
    const float cc = clip ? clip[0] : 1.f;
    const float step_size = lr / bc1;
    const float decay = 1.f - lr * wd, omb1 = 1.f - b1, omb2 = 1.f - b2;
    // 16-byte vector body (flat shards are 128-byte aligned), scalar tail below
    const bool vec_ok = ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) |
                          reinterpret_cast<uintptr_t>(v)) & 15) == 0 &&
                        (pb == nullptr || (reinterpret_cast<uintptr_t>(pb) & 7) == 0);
    const int64_t n4 = vec_ok ? (n >> 2) : 0;
    for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n4; i += int64_t(gridDim.x) * blockDim.x) {
        const float4 g4 = __ldg(reinterpret_cast<const float4*>(g) + i);
        float4 p4 = reinterpret_cast<float4*>(p)[i];
        float4 m4 = reinterpret_cast<float4*>(m)[i];
        float4 v4 = reinterpret_cast<float4*>(v)[i];
        float* pp = reinterpret_cast<float*>(&p4);
        float* mm = reinterpret_cast<float*>(&m4);
        float* vv = reinterpret_cast<float*>(&v4);
        const float* gg = reinterpret_cast<const float*>(&g4);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float gi = gg[j] * cc;
            float pi = pp[j] * decay;
            const float mi = b1 * mm[j] + omb1 * gi;
            const float vi = b2 * vv[j] + omb2 * gi * gi;
            const float denom = sqrtf(vi) / bc2_sqrt + eps;
            pi -= step_size * (mi / denom);
            pp[j] = pi;
            mm[j] = mi;
            vv[j] = vi;
        }
        reinterpret_cast<float4*>(p)[i] = p4;
        reinterpret_cast<float4*>(m)[i] = m4;
        reinterpret_cast<float4*>(v)[i] = v4;
        if (pb) {
            uint2 o;
            o.x = pack_bf16(p4.x, p4.y);
            o.y = pack_bf16(p4.z, p4.w);
            reinterpret_cast<uint2*>(pb)[i] = o;
        }
    }
    for (int64_t i = (n4 << 2) + int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
         i += int64_t(gridDim.x) * blockDim.x) {
        const float gi = g[i] * cc;
        float pi = p[i] * (1.f - lr * wd);
        const float mi = b1 * m[i] + (1.f - b1) * gi;
        const float vi = b2 * v[i] + (1.f - b2) * gi * gi;
        const float denom = sqrtf(vi) / bc2_sqrt + eps;
        pi -= step_size * (mi / denom);
        p[i] = pi;
        m[i] = mi;
        v[i] = vi;
        if (pb) pb[i] = __float2bfloat16_rn(pi);
    }
}

__global__ void __launch_bounds__(kThreads)
    cast_f32_bf16_kernel(const float* __restrict__ s, __nv_bfloat16* __restrict__ d, int64_t n) {
    for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += int64_t(gridDim.x) * blockDim.x)
        d[i] = __float2bfloat16_rn(s[i]);
}
__global__ void __launch_bounds__(kThreads)
    accum_bf16_f32_kernel(const __nv_bfloat16* __restrict__ s, float* __restrict__ d, float scale, int64_t n) {
    for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += int64_t(gridDim.x) * blockDim.x)
        d[i] += scale * __bfloat162float(s[i]);
}

inline int grid_for(int64_t work_items, int per_block) {
    int64_t b = (work_items + per_block - 1) / per_block;
    const int64_t cap = int64_t(dolo_num_sms()) * 8;
    if (b > cap) b = cap;
    if (b < 1) b = 1;
    return int(b);
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace

// ==========================================================================================
// C ABI
// ==========================================================================================
extern "C" int dolomite_b200_rmsnorm_fwd(const void* x, const void* w, void* y, float* rstd, int64_t T, int H,
                                         float eps, void* stream) {
    DOLO_REQUIRE(H > 0 && H % 8 == 0, "rmsnorm: H=%d must be a positive multiple of 8", H);
    DOLO_REQUIRE(H <= 8 * kThreads * 8, "rmsnorm: H=%d too large (max %d)", H, 8 * kThreads * 8);
    DOLO_REQUIRE(aligned16(x) && aligned16(w) && aligned16(y), "rmsnorm: pointers must be 16-byte aligned");
    if (T == 0) return DOLO_OK;
    const int H8 = H / 8;
    const int nv = (H8 + kThreads - 1) / kThreads;
    const int grid = int(T < int64_t(dolo_num_sms()) * 16 ? T : int64_t(dolo_num_sms()) * 16);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    auto X = static_cast<const uint4*>(x);
    auto W = static_cast<const uint4*>(w);
    auto Y = static_cast<uint4*>(y);
    const float inv_h = 1.f / float(H);
    if (H8 <= 16 * 32 && T >= 64) {  // one warp per row
        const int64_t want = (T + kWarpRowThreads / 32 - 1) / (kWarpRowThreads / 32);
        const int wgrid = int(want < (1ll << 30) ? want : (1ll << 30));
        const int nvw = (H8 + 31) / 32;
        if (nvw <= 4) rmsnorm_fwd_warp_kernel<4><<<wgrid, kWarpRowThreads, 0, st>>>(X, W, Y, rstd, T, H8, eps, inv_h);
        else if (nvw <= 8) rmsnorm_fwd_warp_kernel<8><<<wgrid, kWarpRowThreads, 0, st>>>(X, W, Y, rstd, T, H8, eps, inv_h);
        else if (nvw <= 10) rmsnorm_fwd_warp_kernel<10><<<wgrid, kWarpRowThreads, 0, st>>>(X, W, Y, rstd, T, H8, eps, inv_h);
        else rmsnorm_fwd_warp_kernel<16><<<wgrid, kWarpRowThreads, 0, st>>>(X, W, Y, rstd, T, H8, eps, inv_h);
        DOLO_LAUNCH_OK("rmsnorm_fwd");
        return DOLO_OK;
    }
    switch (nv) {
        case 1: rmsnorm_fwd_kernel<1><<<grid, kThreads, 0, st>>>(X, W, Y, rstd, T, H8, eps, inv_h); break;
        case 2: rmsnorm_fwd_kernel<2><<<grid, kThreads, 0, st>>>(X, W, Y, rstd, T, H8, eps, inv_h); break;
        case 3:
        case 4: rmsnorm_fwd_kernel<4><<<grid, kThreads, 0, st>>>(X, W, Y, rstd, T, H8, eps, inv_h); break;
        default: rmsnorm_fwd_kernel<8><<<grid, kThreads, 0, st>>>(X, W, Y, rstd, T, H8, eps, inv_h); break;
    }
    DOLO_LAUNCH_OK("rmsnorm_fwd");
    return DOLO_OK;
}

// Each block alternates a load phase, a block reduction and a store phase, so it takes several independent blocks per SM to
// keep HBM requests in flight.  The RMSNorm backward sizes its blocks to the row (H = 2560: 160 threads x 2 vectors -- with 256
// threads 192 of them held one vector in two vectors' worth of registers), which fits 6 blocks of 64 registers per SM.
static int rmsnorm_bwd_parts() { return dolo_num_sms() * 6; }

extern "C" int64_t dolomite_b200_rmsnorm_bwd_workspace_bytes(int H) {
    return int64_t(rmsnorm_bwd_parts()) * H * sizeof(float);
}

extern "C" int dolomite_b200_rmsnorm_bwd(const void* dy, const void* x, const void* w, const float* rstd,
                                         const void* dx_add, void* dx, float* dw_accum, void* workspace, int64_t T,
                                         int H, void* stream) {
    DOLO_REQUIRE(H > 0 && H % 8 == 0, "rmsnorm_bwd: H=%d must be a positive multiple of 8", H);
    DOLO_REQUIRE(H <= 8 * kThreads * 8, "rmsnorm_bwd: H=%d too large", H);
    DOLO_REQUIRE(aligned16(dy) && aligned16(x) && aligned16(w) && aligned16(dx) && aligned16(workspace) &&
                     aligned16(dx_add),
                 "rmsnorm_bwd: pointers must be 16-byte aligned");
    if (T == 0) return DOLO_OK;
    const int H8 = H / 8;
    const int nv = (H8 + kThreads - 1) / kThreads;
    int parts = rmsnorm_bwd_parts();
    if (T < parts) parts = int(T);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    auto DY = static_cast<const uint4*>(dy);
    auto X = static_cast<const uint4*>(x);
    auto W = static_cast<const uint4*>(w);
    auto DA = static_cast<const uint4*>(dx_add);
    auto DX = static_cast<uint4*>(dx);
    auto WS = static_cast<float*>(workspace);
    const float inv_h = 1.f / float(H);
    const int nvk = nv <= 2 ? nv : (nv <= 4 ? 4 : 8);                    // vectors per thread of the instantiation used
    int threads = ((H8 + nvk - 1) / nvk + 31) / 32 * 32;                  // just enough warps for the row
    if (threads > kThreads) threads = kThreads;
    switch (nvk) {
        case 1: rmsnorm_bwd_kernel<1><<<parts, threads, 0, st>>>(DY, X, W, rstd, DA, DX, WS, T, H8, inv_h); break;
        case 2: rmsnorm_bwd_kernel<2><<<parts, threads, 0, st>>>(DY, X, W, rstd, DA, DX, WS, T, H8, inv_h); break;
        case 4: rmsnorm_bwd_kernel<4><<<parts, threads, 0, st>>>(DY, X, W, rstd, DA, DX, WS, T, H8, inv_h); break;
        default: rmsnorm_bwd_kernel<8><<<parts, threads, 0, st>>>(DY, X, W, rstd, DA, DX, WS, T, H8, inv_h); break;
    }
    DOLO_LAUNCH_OK("rmsnorm_bwd");
    if (dw_accum != nullptr) {
        reduce_partials_kernel<<<(H + 31) / 32, 256, 0, st>>>(WS, dw_accum, parts, H, H);
        DOLO_LAUNCH_OK("rmsnorm_bwd_reduce");
    }
    return DOLO_OK;
}

extern "C" int dolomite_b200_layernorm_fwd(const void* x, const void* w, const void* b, void* y, float* mean, float* rstd,
                                           int64_t T, int H, float eps, void* stream) {
    DOLO_REQUIRE(H > 0 && H % 8 == 0, "layernorm: H=%d must be a positive multiple of 8", H);
    DOLO_REQUIRE(H <= 8 * kThreads * 8, "layernorm: H=%d too large (max %d)", H, 8 * kThreads * 8);
    DOLO_REQUIRE(aligned16(x) && aligned16(w) && aligned16(y) && aligned16(b), "layernorm: pointers must be 16-byte aligned");
    if (T == 0) return DOLO_OK;
    const int H8 = H / 8;
    const int nv = (H8 + kThreads - 1) / kThreads;
    const int grid = int(T < int64_t(dolo_num_sms()) * 16 ? T : int64_t(dolo_num_sms()) * 16);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    auto X = static_cast<const uint4*>(x);
    auto W = static_cast<const uint4*>(w);
    auto B = static_cast<const uint4*>(b);
    auto Y = static_cast<uint4*>(y);
    const float inv_h = 1.f / float(H);
    switch (nv) {
        case 1: layernorm_fwd_kernel<1><<<grid, kThreads, 0, st>>>(X, W, B, Y, mean, rstd, T, H8, eps, inv_h); break;
        case 2: layernorm_fwd_kernel<2><<<grid, kThreads, 0, st>>>(X, W, B, Y, mean, rstd, T, H8, eps, inv_h); break;
        case 3:
        case 4: layernorm_fwd_kernel<4><<<grid, kThreads, 0, st>>>(X, W, B, Y, mean, rstd, T, H8, eps, inv_h); break;
        default: layernorm_fwd_kernel<8><<<grid, kThreads, 0, st>>>(X, W, B, Y, mean, rstd, T, H8, eps, inv_h); break;
    }
    DOLO_LAUNCH_OK("layernorm_fwd");
    return DOLO_OK;
}

extern "C" int64_t dolomite_b200_layernorm_bwd_workspace_bytes(int H) {
    return int64_t(rmsnorm_bwd_parts()) * 2 * H * sizeof(float);
}

extern "C" int dolomite_b200_layernorm_bwd(const void* dy, const void* x, const void* w, const float* mean,
                                           const float* rstd, const void* dx_add, void* dx, float* dw_accum,
                                           float* db_accum, void* workspace, int64_t T, int H, void* stream) {
    DOLO_REQUIRE(H > 0 && H % 8 == 0, "layernorm_bwd: H=%d must be a positive multiple of 8", H);
    DOLO_REQUIRE(H <= 8 * kThreads * 8, "layernorm_bwd: H=%d too large", H);
    DOLO_REQUIRE(aligned16(dy) && aligned16(x) && aligned16(w) && aligned16(dx) && aligned16(workspace) &&
                     aligned16(dx_add),
                 "layernorm_bwd: pointers must be 16-byte aligned");
    if (T == 0) return DOLO_OK;
    const int H8 = H / 8;
    const int nv = (H8 + kThreads - 1) / kThreads;
    int parts = rmsnorm_bwd_parts();
    if (T < parts) parts = int(T);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    auto DY = static_cast<const uint4*>(dy);
    auto X = static_cast<const uint4*>(x);
    auto W = static_cast<const uint4*>(w);
    auto DA = static_cast<const uint4*>(dx_add);
    auto DX = static_cast<uint4*>(dx);
    auto WS = static_cast<float*>(workspace);
    const float inv_h = 1.f / float(H);
    switch (nv) {
        case 1: layernorm_bwd_kernel<1><<<parts, kThreads, 0, st>>>(DY, X, W, mean, rstd, DA, DX, WS, T, H8, inv_h); break;
        case 2: layernorm_bwd_kernel<2><<<parts, kThreads, 0, st>>>(DY, X, W, mean, rstd, DA, DX, WS, T, H8, inv_h); break;
        case 3:
        case 4: layernorm_bwd_kernel<4><<<parts, kThreads, 0, st>>>(DY, X, W, mean, rstd, DA, DX, WS, T, H8, inv_h); break;
        default: layernorm_bwd_kernel<8><<<parts, kThreads, 0, st>>>(DY, X, W, mean, rstd, DA, DX, WS, T, H8, inv_h); break;
    }
    DOLO_LAUNCH_OK("layernorm_bwd");
    if (dw_accum != nullptr) {
        reduce_partials_kernel<<<(H + 31) / 32, 256, 0, st>>>(WS, dw_accum, parts, H, 2 * H);
        DOLO_LAUNCH_OK("layernorm_bwd_reduce_w");
    }
    if (db_accum != nullptr) {
        reduce_partials_kernel<<<(H + 31) / 32, 256, 0, st>>>(WS + H, db_accum, parts, H, 2 * H);
        DOLO_LAUNCH_OK("layernorm_bwd_reduce_b");
    }
    return DOLO_OK;
}

extern "C" int dolomite_b200_rope_qk_inplace(void* qkv, int64_t row_stride, int64_t T, int n_groups, int q_per_group,
                                             int head_dim, const void* cos_table, const void* sin_table,
                                             const void* position_ids, int position_ids_is_int64, int64_t n_positions,
                                             int inverse, void* stream) {
    DOLO_REQUIRE(head_dim > 0 && head_dim % 16 == 0, "rope: head_dim=%d must be a multiple of 16", head_dim);
    DOLO_REQUIRE(row_stride % 8 == 0 && aligned16(qkv) && aligned16(cos_table) && aligned16(sin_table),
                 "rope: 16-byte alignment required (row_stride %lld)", (long long)row_stride);
    DOLO_REQUIRE(int64_t(n_groups) * (q_per_group + 2) * head_dim <= row_stride, "rope: slot layout exceeds row stride");
    DOLO_REQUIRE(n_positions > 0, "rope: empty cos/sin table");
    if (T == 0) return DOLO_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int items = n_groups * (q_per_group + 1) * (head_dim / 16);
    const int threads = items >= 1024 ? 1024 : ((items + 31) / 32) * 32;
    const int64_t want = int64_t(dolo_num_sms()) * (2048 / threads);
    const int grid = int(T < want ? T : want);
    const float sgn = inverse ? -1.f : 1.f;
    auto Q = static_cast<__nv_bfloat16*>(qkv);
    auto C = static_cast<const __nv_bfloat16*>(cos_table);
    auto S = static_cast<const __nv_bfloat16*>(sin_table);
    if (position_ids_is_int64) {
        auto P = static_cast<const int64_t*>(position_ids);
        if (threads <= 512)
            rope_kernel<int64_t, 512><<<grid, threads, 0, st>>>(Q, row_stride, T, n_groups, q_per_group, head_dim, C, S, P, n_positions, sgn);
        else
            rope_kernel<int64_t, 1024><<<grid, threads, 0, st>>>(Q, row_stride, T, n_groups, q_per_group, head_dim, C, S, P, n_positions, sgn);
    } else {
        auto P = static_cast<const int32_t*>(position_ids);
        if (threads <= 512)
            rope_kernel<int32_t, 512><<<grid, threads, 0, st>>>(Q, row_stride, T, n_groups, q_per_group, head_dim, C, S, P, n_positions, sgn);
        else
            rope_kernel<int32_t, 1024><<<grid, threads, 0, st>>>(Q, row_stride, T, n_groups, q_per_group, head_dim, C, S, P, n_positions, sgn);
    }
    DOLO_LAUNCH_OK("rope");
    return DOLO_OK;
}

namespace {

// fn(Op{}) with the functor of activation `id`; false for an unknown id
template <class Fn>
bool visit_act(int id, Fn&& fn) {
    switch (id) {
        case DOLO_ACT_CELU:
        case DOLO_ACT_ELU: fn(act::Elu{}); return true;
        case DOLO_ACT_GELU: fn(act::Gelu{}); return true;
        case DOLO_ACT_GELU_TANH: fn(act::GeluTanh{}); return true;
        case DOLO_ACT_SELU: fn(act::Selu{}); return true;
        case DOLO_ACT_HARDSHRINK: fn(act::HardShrink{}); return true;
        case DOLO_ACT_HARDSIGMOID: fn(act::HardSigmoid{}); return true;
        case DOLO_ACT_HARDSWISH: fn(act::HardSwish{}); return true;
        case DOLO_ACT_HARDTANH: fn(act::HardTanh{}); return true;
        case DOLO_ACT_LAPLACE: fn(act::Laplace{}); return true;
        case DOLO_ACT_LEAKY_RELU: fn(act::LeakyRelu{}); return true;
        case DOLO_ACT_LOG_SIGMOID: fn(act::LogSigmoid{}); return true;
        case DOLO_ACT_MISH: fn(act::Mish{}); return true;
        case DOLO_ACT_RELU: fn(act::Relu{}); return true;
        case DOLO_ACT_RELU2: fn(act::Relu2{}); return true;
        case DOLO_ACT_RELU6: fn(act::Relu6{}); return true;
        case DOLO_ACT_SIGMOID: fn(act::Sigmoid{}); return true;
        case DOLO_ACT_SILU: fn(act::Silu{}); return true;
        case DOLO_ACT_SOFTPLUS: fn(act::Softplus{}); return true;
        case DOLO_ACT_SOFTSHRINK: fn(act::SoftShrink{}); return true;
        case DOLO_ACT_SOFTSIGN: fn(act::SoftSign{}); return true;
        case DOLO_ACT_TANH: fn(act::Tanh{}); return true;
        case DOLO_ACT_TANHSHRINK: fn(act::TanhShrink{}); return true;
        default: return false;
    }
}

template <class Op>
void launch_act_fwd(int form, const void* x, void* y, int64_t T, int64_t F8, cudaStream_t st) {
    auto X = static_cast<const uint4*>(x);
    auto Y = static_cast<uint4*>(y);
    const int grid = grid_for(T * F8, kThreads);
    if (form == DOLO_ACT_PLAIN) {
        act_fwd_kernel<Op, DOLO_ACT_PLAIN><<<grid, kThreads, 0, st>>>(X, Y, T, F8);
    } else if (form == DOLO_ACT_GLU) {
        act_fwd_kernel<Op, DOLO_ACT_GLU><<<grid, kThreads, 0, st>>>(X, Y, T, F8);
    } else if constexpr (std::is_same_v<Op, act::Sigmoid>) {  // torch's fused glu exists for the sigmoid only
        act_fwd_kernel<Op, DOLO_ACT_SIGMOID_GLU><<<grid, kThreads, 0, st>>>(X, Y, T, F8);
    }
}

// seg / segments: segment table of the rows (NULL: the dense launch, one segment of T rows); dbias_seg_stride floats
// between the bias-gradient rows of consecutive segments
template <class Op, bool Glu>
cudaError_t launch_act_bwd_form(const void* dy, const void* x, void* dx, float* dbias, int64_t T, int64_t F8,
                                const int* seg, int segments, int64_t dbias_seg_stride, cudaStream_t st) {
    auto DY = static_cast<const uint4*>(dy);
    auto X = static_cast<const uint4*>(x);
    auto DX = static_cast<uint4*>(dx);
    if (dbias == nullptr) {
        act_bwd_kernel<Op, Glu><<<grid_for(T * F8, kThreads), kThreads, 0, st>>>(DY, X, DX, T, F8);
        return cudaGetLastError();
    }
    const int col_tiles = int((F8 + 31) / 32);
    const int rows_per_block = int((T + kColsumCluster - 1) / kColsumCluster);  // one cluster of row splits per column tile
    return cudaError_t(launch_row_cluster(act_bwd_bias_kernel<Op, Glu>, col_tiles, segments, st, DY, X, DX, dbias, T, F8,
                                          rows_per_block, seg, dbias_seg_stride));
}

int check_act(const char* what, int act_id, int form, int64_t F) {
    DOLO_REQUIRE(act_id >= 0 && act_id < DOLO_ACT_COUNT, "%s: unknown activation id %d", what, act_id);
    DOLO_REQUIRE(form == DOLO_ACT_PLAIN || form == DOLO_ACT_GLU || (form == DOLO_ACT_SIGMOID_GLU && act_id == DOLO_ACT_SIGMOID),
                 "%s: form %d is not defined for activation id %d", what, form, act_id);
    DOLO_REQUIRE(F > 0 && F % 8 == 0, "%s: F=%lld must be a positive multiple of 8", what, (long long)F);
    return DOLO_OK;
}

}  // namespace

extern "C" int dolomite_b200_act_fwd(int act_id, int form, const void* x, void* y, int64_t T, int64_t F, void* stream) {
    if (const int rc = check_act("act_fwd", act_id, form, F)) return rc;
    DOLO_REQUIRE(aligned16(x) && aligned16(y), "act_fwd: pointers must be 16-byte aligned");
    if (T == 0) return DOLO_OK;
    visit_act(act_id, [&](auto op) {
        launch_act_fwd<decltype(op)>(form, x, y, T, F / 8, static_cast<cudaStream_t>(stream));
    });
    DOLO_LAUNCH_OK("act_fwd");
    return DOLO_OK;
}

extern "C" int dolomite_b200_act_bwd(int act_id, int form, const void* dy, const void* x, void* dx, float* dbias_accum,
                                     int64_t T, int64_t F, void* stream) {
    if (const int rc = check_act("act_bwd", act_id, form, F)) return rc;
    DOLO_REQUIRE(aligned16(x) && aligned16(dy) && aligned16(dx), "act_bwd: pointers must be 16-byte aligned");
    if (T == 0) return DOLO_OK;
    cudaError_t e = cudaSuccess;
    visit_act(act_id, [&](auto op) {
        using Op = decltype(op);
        const cudaStream_t st = static_cast<cudaStream_t>(stream);
        e = form == DOLO_ACT_PLAIN ? launch_act_bwd_form<Op, false>(dy, x, dx, dbias_accum, T, F / 8, nullptr, 1, 0, st)
                                   : launch_act_bwd_form<Op, true>(dy, x, dx, dbias_accum, T, F / 8, nullptr, 1, 0, st);
    });
    DOLO_CUDA_OK(e);
    return DOLO_OK;
}

extern "C" int dolomite_b200_act_bwd_segmented(int act_id, int form, const void* dy, const void* x, void* dx,
                                               float* dbias_accum, int64_t ld_dbias, int64_t F,
                                               const int32_t* seg_offsets, int num_segments, void* stream) {
    if (const int rc = check_act("act_bwd_segmented", act_id, form, F)) return rc;
    DOLO_REQUIRE(aligned16(x) && aligned16(dy) && aligned16(dx), "act_bwd_segmented: pointers must be 16-byte aligned");
    DOLO_REQUIRE(dbias_accum != nullptr && seg_offsets != nullptr && num_segments > 0 && num_segments <= 65535,
                 "act_bwd_segmented: bias gradient, segment table and 1..65535 segments needed");
    const int64_t fc_out = form == DOLO_ACT_PLAIN ? F : 2 * F;
    DOLO_REQUIRE(ld_dbias >= fc_out, "act_bwd_segmented: ld_dbias=%lld < %lld columns", (long long)ld_dbias,
                 (long long)fc_out);
    cudaError_t e = cudaSuccess;
    visit_act(act_id, [&](auto op) {
        using Op = decltype(op);
        const cudaStream_t st = static_cast<cudaStream_t>(stream);
        e = form == DOLO_ACT_PLAIN
                ? launch_act_bwd_form<Op, false>(dy, x, dx, dbias_accum, 0, F / 8, seg_offsets, num_segments, ld_dbias, st)
                : launch_act_bwd_form<Op, true>(dy, x, dx, dbias_accum, 0, F / 8, seg_offsets, num_segments, ld_dbias, st);
    });
    DOLO_CUDA_OK(e);
    return DOLO_OK;
}

// the SwiGLU / tanh-GELU entry points of ABI version 1
extern "C" int dolomite_b200_gelu_fwd(const void* x, void* y, int64_t n, void* stream) {
    DOLO_REQUIRE(n % 8 == 0 && aligned16(x) && aligned16(y), "gelu: n must be a multiple of 8 and pointers 16-byte aligned");
    if (n == 0) return DOLO_OK;
    launch_act_fwd<act::GeluTanh>(DOLO_ACT_PLAIN, x, y, n / 8, 1, static_cast<cudaStream_t>(stream));
    DOLO_LAUNCH_OK("gelu_fwd");
    return DOLO_OK;
}

extern "C" int dolomite_b200_gelu_bwd(const void* dy, const void* x, void* dx, float* dbias_accum, int64_t T, int64_t F,
                                      void* stream) {
    return dolomite_b200_act_bwd(DOLO_ACT_GELU_TANH, DOLO_ACT_PLAIN, dy, x, dx, dbias_accum, T, F, stream);
}

extern "C" int dolomite_b200_swiglu_fwd(const void* x, void* y, int64_t T, int64_t F, void* stream) {
    return dolomite_b200_act_fwd(DOLO_ACT_SILU, DOLO_ACT_GLU, x, y, T, F, stream);
}

extern "C" int dolomite_b200_swiglu_bwd(const void* dy, const void* x, void* dx, int64_t T, int64_t F, void* stream) {
    return dolomite_b200_act_bwd(DOLO_ACT_SILU, DOLO_ACT_GLU, dy, x, dx, nullptr, T, F, stream);
}

extern "C" int dolomite_b200_swiglu_bwd_bias(const void* dy, const void* x, void* dx, float* dbias_accum, int64_t T,
                                             int64_t F, void* stream) {
    DOLO_REQUIRE(dbias_accum != nullptr, "swiglu_bwd_bias: bias gradient buffer is null");
    return dolomite_b200_act_bwd(DOLO_ACT_SILU, DOLO_ACT_GLU, dy, x, dx, dbias_accum, T, F, stream);
}

extern "C" int dolomite_b200_embedding_fwd(const int64_t* ids, const void* wte, void* out, int64_t T, int H, int64_t V,
                                           float scale, void* stream) {
    DOLO_REQUIRE(H > 0 && H % 8 == 0, "embedding: H=%d must be a multiple of 8", H);
    DOLO_REQUIRE(aligned16(wte) && aligned16(out), "embedding: pointers must be 16-byte aligned");
    if (T == 0) return DOLO_OK;
    const int grid = int(T < int64_t(dolo_num_sms()) * 16 ? T : int64_t(dolo_num_sms()) * 16);
    embedding_fwd_kernel<<<grid, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
        ids, static_cast<const uint4*>(wte), static_cast<uint4*>(out), T, H / 8, V, scale, scale != 1.f);
    DOLO_LAUNCH_OK("embedding_fwd");
    return DOLO_OK;
}

extern "C" int dolomite_b200_embedding_fwd_neft(const int64_t* ids, const void* wte, void* out, int64_t T, int H, int64_t V,
                                                uint32_t key0, uint32_t key1, float mag, void* stream) {
    DOLO_REQUIRE(H > 0 && H % 8 == 0, "embedding_fwd_neft: H=%d must be a multiple of 8", H);
    DOLO_REQUIRE(aligned16(wte) && aligned16(out), "embedding_fwd_neft: pointers must be 16-byte aligned");
    DOLO_REQUIRE(mag > 0.f && mag < 1e30f, "embedding_fwd_neft: mag=%g must be positive and finite", double(mag));
    if (T == 0) return DOLO_OK;
    // the bounds and the range as torch's uniform_kernel forms them for a bf16 tensor
    const float from = __bfloat162float(__float2bfloat16_rn(-mag));
    const float to = __bfloat162float(__float2bfloat16_rn(mag));
    const float range = __bfloat162float(__float2bfloat16_rn(to - from));
    const int grid = int(T < int64_t(dolo_num_sms()) * 16 ? T : int64_t(dolo_num_sms()) * 16);
    embedding_fwd_neft_kernel<<<grid, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
        ids, static_cast<const uint4*>(wte), static_cast<uint4*>(out), T, H / 8, V, key0, key1, from, to, range);
    DOLO_LAUNCH_OK("embedding_fwd_neft");
    return DOLO_OK;
}

extern "C" int dolomite_b200_embedding_bwd(const int64_t* ids, const void* dout, float* dwte, int64_t T, int H,
                                           int64_t V, float scale, void* stream) {
    DOLO_REQUIRE(H > 0 && H % 8 == 0, "embedding_bwd: H=%d must be a multiple of 8", H);
    DOLO_REQUIRE(aligned16(dout) && aligned16(dwte), "embedding_bwd: pointers must be 16-byte aligned");  // dwte: float4
    if (T == 0) return DOLO_OK;
    DOLO_REQUIRE(T < (int64_t(1) << 36), "embedding_bwd: T too large");
    const unsigned grid = unsigned((T + kThreads / 32 - 1) / (kThreads / 32));  // one warp per token
    embedding_bwd_kernel<<<grid, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
        ids, static_cast<const uint4*>(dout), dwte, T, H / 8, V, scale);
    DOLO_LAUNCH_OK("embedding_bwd");
    return DOLO_OK;
}

extern "C" int dolomite_b200_cross_entropy_count(const int64_t* labels, int64_t T, int64_t ignore_index, float* scratch,
                                                 void* stream) {
    ce_count_kernel<<<1, 1024, 0, static_cast<cudaStream_t>(stream)>>>(labels, T, ignore_index, scratch);
    DOLO_LAUNCH_OK("ce_count");
    return DOLO_OK;
}

extern "C" int dolomite_b200_cross_entropy_rows(const void* logits, int64_t ldl, const int64_t* labels, void* dlogits,
                                                float* loss_per_token, const float* scratch, int64_t T, int64_t V,
                                                int64_t ignore_index, float logit_scale, float grad_scale, void* stream) {
    DOLO_REQUIRE(V > 0 && ldl % 8 == 0 && ldl >= V,
                 "cross_entropy: V=%lld must be >= 1 and ld=%lld a multiple of 8 and >= V", (long long)V, (long long)ldl);
    DOLO_REQUIRE(aligned16(logits) && aligned16(dlogits), "cross_entropy: pointers must be 16-byte aligned");
    if (T == 0) return DOLO_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    // vectors per thread with 256 threads and the whole row in ONE CTA; wider rows are split over a 2- or 4-CTA cluster
    const int64_t V8 = (V + 7) / 8;
    const int64_t nv1 = (V8 + kCeThreads - 1) / kCeThreads;
#define DOLO_CE(NV, SPLIT)                                                                                             \
    return V % 8 ? launch_ce_rows<NV, SPLIT, true>(logits, ldl, labels, dlogits, loss_per_token, scratch, T, V,      \
                                                   ignore_index, logit_scale, grad_scale, st)                         \
                 : launch_ce_rows<NV, SPLIT, false>(logits, ldl, labels, dlogits, loss_per_token, scratch, T, V,     \
                                                    ignore_index, logit_scale, grad_scale, st)
    if (nv1 <= 4) DOLO_CE(4, 1);
    if (nv1 <= 8) DOLO_CE(8, 1);
    if (nv1 <= 16) DOLO_CE(16, 1);
    // one CTA per row whenever it fits: the cluster barrier costs a GPU-scope fence per use.  The masked last vector of an
    // odd width pushes the 24-vector instance to 632 bytes of spill loads per thread, so such rows take the 2-CTA cluster.
    if (nv1 <= 24 && V % 8 == 0)
        return launch_ce_rows<24, 1, false>(logits, ldl, labels, dlogits, loss_per_token, scratch, T, V, ignore_index,
                                            logit_scale, grad_scale, st);
    if (nv1 <= 32) DOLO_CE(16, 2);
    if (nv1 <= 48) DOLO_CE(12, 4);
    if (nv1 <= 64) DOLO_CE(16, 4);
#undef DOLO_CE
    return dolo_set_error("cross_entropy: vocabulary %lld exceeds the 131072 columns one 4-CTA cluster holds", (long long)V);
}

extern "C" int dolomite_b200_cross_entropy_mean(const float* loss_per_token, int64_t T, const float* scratch,
                                                float* loss_mean, void* stream) {
    ce_mean_kernel<<<1, 1024, 0, static_cast<cudaStream_t>(stream)>>>(loss_per_token, T, scratch, loss_mean);
    DOLO_LAUNCH_OK("ce_mean");
    return DOLO_OK;
}

extern "C" int dolomite_b200_cross_entropy_fwd_bwd(const void* logits, int64_t ldl, const int64_t* labels,
                                                   void* dlogits, float* loss_per_token, float* loss_mean,
                                                   float* scratch, int64_t T, int64_t V, int64_t ignore_index,
                                                   float logit_scale, float grad_scale, void* stream) {
    int rc = dolomite_b200_cross_entropy_count(labels, T, ignore_index, scratch, stream);
    if (rc) return rc;
    rc = dolomite_b200_cross_entropy_rows(logits, ldl, labels, dlogits, loss_per_token, scratch, T, V, ignore_index,
                                          logit_scale, grad_scale, stream);
    if (rc) return rc;
    return dolomite_b200_cross_entropy_mean(loss_per_token, T, scratch, loss_mean, stream);
}

extern "C" int dolomite_b200_colsum_accum(const void* x, int64_t ldx, float* out, int64_t T, int64_t N, float scale,
                                          void* stream) {
    DOLO_REQUIRE(N > 0 && N % 8 == 0 && ldx % 8 == 0, "colsum: N=%lld / ld=%lld must be multiples of 8", (long long)N,
                 (long long)ldx);
    DOLO_REQUIRE(aligned16(x), "colsum: pointer must be 16-byte aligned");
    if (T == 0) return DOLO_OK;
    const int col_tiles = int((N + 255) / 256);
    const int rows_per_block = int((T + kColsumCluster - 1) / kColsumCluster);  // one cluster of row splits per column tile
    DOLO_CUDA_OK(cudaError_t(launch_row_cluster(colsum_kernel, col_tiles, 1, static_cast<cudaStream_t>(stream),
                                                static_cast<const __nv_bfloat16*>(x), ldx, out, T, N, rows_per_block,
                                                scale, static_cast<const int*>(nullptr), int64_t(0))));
    return DOLO_OK;
}

extern "C" int dolomite_b200_colsum_accum_segmented(const void* x, int64_t ldx, float* out, int64_t ld_out, int64_t N,
                                                    const int32_t* seg_offsets, int num_segments, float scale,
                                                    void* stream) {
    DOLO_REQUIRE(N > 0 && N % 8 == 0 && ldx % 8 == 0, "colsum_segmented: N=%lld / ld=%lld must be multiples of 8",
                 (long long)N, (long long)ldx);
    DOLO_REQUIRE(aligned16(x), "colsum_segmented: pointer must be 16-byte aligned");
    DOLO_REQUIRE(seg_offsets != nullptr && num_segments > 0 && num_segments <= 65535 && ld_out >= N,
                 "colsum_segmented: segment table, 1..65535 segments and ld_out >= N needed");
    const int col_tiles = int((N + 255) / 256);
    DOLO_CUDA_OK(cudaError_t(launch_row_cluster(colsum_kernel, col_tiles, num_segments, static_cast<cudaStream_t>(stream),
                                                static_cast<const __nv_bfloat16*>(x), ldx, out, int64_t(0), N, 0, scale,
                                                static_cast<const int*>(seg_offsets), ld_out)));
    return DOLO_OK;
}

__global__ void __launch_bounds__(256) scale_by_dev_scalar_kernel(uint4* __restrict__ x, int64_t n8,
                                                                  const float* __restrict__ scale) {
    const float s = scale[0];
    if (s == 1.f) return;
    for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n8; i += int64_t(gridDim.x) * blockDim.x) {
        uint4 v = x[i];
        v.x = dolo::pack_bf16(dolo::bf16_lo(v.x) * s, dolo::bf16_hi(v.x) * s);
        v.y = dolo::pack_bf16(dolo::bf16_lo(v.y) * s, dolo::bf16_hi(v.y) * s);
        v.z = dolo::pack_bf16(dolo::bf16_lo(v.z) * s, dolo::bf16_hi(v.z) * s);
        v.w = dolo::pack_bf16(dolo::bf16_lo(v.w) * s, dolo::bf16_hi(v.w) * s);
        x[i] = v;
    }
}

extern "C" int dolomite_b200_scale_bf16_by_device_scalar(void* x, int64_t n, const float* scale, void* stream) {
    DOLO_REQUIRE(n % 8 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0, "scale_bf16: n %% 8 and 16-byte alignment required");
    if (n == 0) return DOLO_OK;
    int64_t blocks = (n / 8 + 255) / 256;
    const int64_t cap = int64_t(dolo_num_sms()) * 8;
    if (blocks > cap) blocks = cap;
    scale_by_dev_scalar_kernel<<<(unsigned)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<uint4*>(x), n / 8, scale);
    DOLO_LAUNCH_OK("scale_bf16_by_device_scalar");
    return DOLO_OK;
}

extern "C" int dolomite_b200_add_scaled(const void* a, const void* b, void* out, float alpha, int64_t n, void* stream) {
    DOLO_REQUIRE(n % 8 == 0, "add_scaled: n=%lld must be a multiple of 8", (long long)n);
    DOLO_REQUIRE(aligned16(a) && aligned16(b) && aligned16(out), "add_scaled: pointers must be 16-byte aligned");
    if (n == 0) return DOLO_OK;
    add_scaled_kernel<<<grid_for(n / 8, kThreads), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const uint4*>(a), static_cast<const uint4*>(b), static_cast<uint4*>(out), alpha, n / 8);
    DOLO_LAUNCH_OK("add_scaled");
    return DOLO_OK;
}

extern "C" int64_t dolomite_b200_sumsq_workspace_bytes(void) { return int64_t(kSumsqBlocks) * 4; }

extern "C" int dolomite_b200_sumsq_accum(const float* g, int64_t n, float* out, void* workspace, void* stream) {
    DOLO_REQUIRE(aligned16(g), "sumsq: pointer must be 16-byte aligned");
    DOLO_REQUIRE(workspace != nullptr && (reinterpret_cast<uintptr_t>(workspace) & 3) == 0, "sumsq: workspace missing or misaligned");
    if (n == 0) return DOLO_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    float* partials = static_cast<float*>(workspace);
    sumsq_partial_kernel<<<kSumsqBlocks, kThreads, 0, st>>>(g, n, partials);
    DOLO_LAUNCH_OK("sumsq_partial");
    sumsq_final_kernel<<<1, kThreads, 0, st>>>(partials, out);
    DOLO_LAUNCH_OK("sumsq_final");
    return DOLO_OK;
}

extern "C" int dolomite_b200_clip_coef(const float* sumsq, float max_norm, float* coef_out, float* norm_out,
                                       void* stream) {
    clip_coef_kernel<<<1, 1, 0, static_cast<cudaStream_t>(stream)>>>(sumsq, max_norm, coef_out, norm_out);
    DOLO_LAUNCH_OK("clip_coef");
    return DOLO_OK;
}

extern "C" int dolomite_b200_adamw_step(float* p, const float* g, float* m, float* v, void* p_bf16, int64_t n, float lr,
                                        float beta1, float beta2, float eps, float weight_decay, int64_t step,
                                        const float* clip_coef, void* stream) {
    DOLO_REQUIRE(step >= 1, "adamw: step must be >= 1 (got %lld)", (long long)step);
    if (n == 0) return DOLO_OK;
    const float bc1 = 1.f - powf(beta1, float(step));
    const float bc2 = 1.f - powf(beta2, float(step));
    adamw_kernel<<<grid_for(n, kThreads), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
        p, g, m, v, static_cast<__nv_bfloat16*>(p_bf16), n, lr, beta1, beta2, eps, weight_decay, bc1, sqrtf(bc2),
        clip_coef);
    DOLO_LAUNCH_OK("adamw");
    return DOLO_OK;
}

extern "C" int dolomite_b200_cast_f32_to_bf16(const float* src, void* dst, int64_t n, void* stream) {
    if (n == 0) return DOLO_OK;
    cast_f32_bf16_kernel<<<grid_for(n, kThreads), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
        src, static_cast<__nv_bfloat16*>(dst), n);
    DOLO_LAUNCH_OK("cast_f32_to_bf16");
    return DOLO_OK;
}

extern "C" int dolomite_b200_accum_bf16_into_f32(const void* src, float* dst, float scale, int64_t n, void* stream) {
    if (n == 0) return DOLO_OK;
    accum_bf16_f32_kernel<<<grid_for(n, kThreads), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const __nv_bfloat16*>(src), dst, scale, n);
    DOLO_LAUNCH_OK("accum_bf16_into_f32");
    return DOLO_OK;
}
