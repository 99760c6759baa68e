// MoE routing / dispatch kernels of the MoEDolomite hot path (reference: moe_dolomite/moe/base.py:108-181 eager
// SparseMoE and moe/scatter.py:109-138 ScatterMoE; third-party scattermoe `flatten_and_sort`,
// `padded_block_indices`, `parallel_linear` semantics per SURVEY.md section 2.3).
//
// Device-side only, no host sync (the eager reference calls .tolist(), moe/base.py:33):
//   route      : top-k on the raw router logits, fp32 softmax over the k selected, per-expert histogram
//   plan       : expert segments padded to 256 rows (two 128-row GEMM tiles) -> offsets, 128-row tile->expert table, row assignment
//   gather     : X_g[row] = x[token(row)] (zero rows for padding) -- operand of the grouped c_fc GEMM
//   combine    : y[t] = sum_j w[t,j] * Y_g[row(t,j)]            -- after the grouped c_proj GEMM
//   backward   : dY_g rows / gate-weight grads, token-sum of dX_g rows, softmax-over-k backward to dense dlogits
// The expert GEMMs themselves are the wgmma GEMM in grouped mode (gemm.cu).
#include "common.cuh"
#include "../../include/dolomite_b200.h"

using namespace dolo;

namespace {

constexpr int MOE_TILE = 128;  // granularity of the tile -> expert table (one entry per 128 grouped rows)
constexpr int MOE_PAD = 256;   // expert segments are padded to 256 rows (a multiple of the 128-row GEMM tile)

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

// Rank of a logit in torch.topk's order as an unsigned key: NaN above everything, then the float order (-inf included,
// -0 equal to +0).  Every logit has a key >= 0x007fffff (that of -inf), so key 0 marks experts that are not candidates
// (chosen already, or lanes past E).
__device__ __forceinline__ uint32_t topk_key(float x) {
    if (x != x) return 0xffffffffu;
    const uint32_t u = __float_as_uint(x + 0.f);  // -0 -> +0
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float topk_value(uint32_t key) {
    return __uint_as_float((key & 0x80000000u) ? (key & 0x7fffffffu) : ~key);
}

// one warp per token.  logits bf16 [T, E]; selects k experts by repeated arg-max of topk_key (ties -> lowest index):
// every logit, -inf and NaN included, can be chosen, so the k chosen experts are distinct and in [0, E) (k <= E).
__global__ void moe_route_kernel(const __nv_bfloat16* __restrict__ logits, int64_t T, int E, int k,
                                 int32_t* __restrict__ sel_idx, float* __restrict__ sel_w,
                                 int32_t* __restrict__ counts) {
    const int64_t t = (int64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (t >= T) return;
    constexpr int MAXE = 8;  // experts per lane -> E <= 256
    uint32_t v[MAXE];
#pragma unroll
    for (int i = 0; i < MAXE; ++i) {
        const int e = lane + i * 32;
        v[i] = e < E ? topk_key(__bfloat162float(logits[t * E + e])) : 0u;
    }
    float chosen_v[8];
    int chosen_e[8];
    for (int j = 0; j < k; ++j) {
        uint32_t best = 0u;
        int be = 0x7fffffff;
#pragma unroll
        for (int i = 0; i < MAXE; ++i) {
            const int e = lane + i * 32;
            if (v[i] > best) { best = v[i]; be = e; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const uint32_t ob = __shfl_xor_sync(0xffffffffu, best, o);
            const int oe = __shfl_xor_sync(0xffffffffu, be, o);
            if (ob > best || (ob == best && oe < be)) { best = ob; be = oe; }
        }
        chosen_v[j] = topk_value(best);
        chosen_e[j] = be;
#pragma unroll
        for (int i = 0; i < MAXE; ++i)
            if (lane + i * 32 == be) v[i] = 0u;
    }
    if (lane == 0) {
        float m = chosen_v[0];
        for (int j = 1; j < k; ++j) m = fmaxf(m, chosen_v[j]);
        float s = 0.f;
        for (int j = 0; j < k; ++j) s += __expf(chosen_v[j] - m);
        for (int j = 0; j < k; ++j) {
            sel_idx[t * k + j] = chosen_e[j];
            sel_w[t * k + j] = __expf(chosen_v[j] - m) / s;
            atomicAdd(counts + chosen_e[j], 1);
        }
    }
}

// single block: padded exclusive scan of the histogram, tile->expert table, cursor reset
__global__ void moe_plan_kernel(const int32_t* __restrict__ counts, int E, int32_t* __restrict__ offsets_padded,
                                int32_t* __restrict__ m_tile_group, int max_tiles, int32_t* __restrict__ cursors) {
    __shared__ int32_t s_off[1025];
    if (threadIdx.x == 0) {
        int acc = 0;
        for (int e = 0; e < E; ++e) {
            s_off[e] = acc;
            acc += (counts[e] + MOE_PAD - 1) / MOE_PAD * MOE_PAD;
        }
        s_off[E] = acc;
    }
    __syncthreads();
    for (int e = threadIdx.x; e <= E; e += blockDim.x) offsets_padded[e] = s_off[e];
    for (int e = threadIdx.x; e < E; e += blockDim.x) cursors[e] = 0;
    for (int i = threadIdx.x; i < max_tiles; i += blockDim.x) {
        const int row = i * MOE_TILE;
        int g = -1;
        if (row < s_off[E]) {
            int lo = 0, hi = E;  // last e with s_off[e] <= row
            while (hi - lo > 1) {
                const int mid = (lo + hi) >> 1;
                if (s_off[mid] <= row) lo = mid; else hi = mid;
            }
            g = lo;
        }
        m_tile_group[i] = g;
    }
}

// Grouped row of every token-slot: expert e's slots take the rows of its segment in slot (= token) order, a stable
// assignment that is the same on every run (an atomic cursor would hand out rows in arrival order).  One block per
// expert scans all slots in chunks of blockDim: ballot + popc give each matching slot its rank inside the chunk.
__global__ void __launch_bounds__(1024)
    moe_assign_kernel(const int32_t* __restrict__ sel_idx, int64_t n_slots, const int32_t* __restrict__ offsets_padded,
                      int32_t* __restrict__ row_of_slot, int32_t* __restrict__ slot_of_row,
                      int32_t* __restrict__ token_of_row, int k) {
    __shared__ int warp_cnt[32];
    const int e = blockIdx.x;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
    int base = offsets_padded[e];
    for (int64_t c0 = 0; c0 < n_slots; c0 += blockDim.x) {
        const int64_t s = c0 + threadIdx.x;
        const bool m = s < n_slots && sel_idx[s] == e;
        const uint32_t bal = __ballot_sync(0xffffffffu, m);
        if (lane == 0) warp_cnt[wid] = __popc(bal);
        __syncthreads();
        int before = 0, total = 0;
        for (int w = 0; w < nw; ++w) {
            before += w < wid ? warp_cnt[w] : 0;
            total += warp_cnt[w];
        }
        if (m) {
            const int row = base + before + __popc(bal & ((1u << lane) - 1u));
            row_of_slot[s] = row;
            slot_of_row[row] = int32_t(s);
            token_of_row[row] = int32_t(s / k);
        }
        base += total;
        __syncthreads();  // warp_cnt is rewritten by the next chunk
    }
}

// X_g[row] = x[slot_of_row[row] / k]  (zeros for padding rows); one warp per row
__global__ void moe_gather_kernel(const uint4* __restrict__ x, uint4* __restrict__ xg,
                                  const int32_t* __restrict__ slot_of_row, const int32_t* __restrict__ offsets_padded,
                                  int E, int k, int H8, int64_t max_rows) {
    const int64_t row = (int64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (row >= max_rows || row >= offsets_padded[E]) return;
    const int slot = slot_of_row[row];
    uint4* dst = xg + row * H8;
    if (slot < 0) {
        for (int i = lane; i < H8; i += 32) dst[i] = make_uint4(0, 0, 0, 0);
    } else {
        const uint4* src = x + int64_t(slot / k) * H8;
        for (int i = lane; i < H8; i += 32) dst[i] = __ldg(src + i);
    }
}

// out[t] = c[t] + alpha * sum_j bf16(w[t,j]) * Y_g[row_of_slot[t*k+j]]     (one warp per token)
__global__ void moe_combine_kernel(const uint4* __restrict__ yg, const int32_t* __restrict__ row_of_slot,
                                   const float* __restrict__ sel_w, const uint4* __restrict__ c, uint4* __restrict__ out,
                                   int64_t T, int k, int H8, float alpha) {
    const int64_t t = (int64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (t >= T) return;
    for (int i = lane; i < H8; i += 32) {
        float acc[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[q] = 0.f;
        for (int j = 0; j < k; ++j) {
            const float w = bf16_round(sel_w[t * k + j]);
            float f[8];
            unpack8(__ldg(yg + int64_t(row_of_slot[t * k + j]) * H8 + i), f);
#pragma unroll
            for (int q = 0; q < 8; ++q) acc[q] += bf16_round(w * f[q]);
        }
        if (c != nullptr) {
            float f[8];
            unpack8(__ldg(c + t * H8 + i), f);
#pragma unroll
            for (int q = 0; q < 8; ++q) acc[q] = f[q] + bf16_round(alpha * bf16_round(acc[q]));
        } else {
#pragma unroll
            for (int q = 0; q < 8; ++q) acc[q] *= alpha;
        }
        out[t * H8 + i] = pack8(acc);
    }
}

// backward of combine: per row, dY_g[row] = alpha * w[slot] * dy[token]; dw[slot] = alpha * <dy[token], Y_g[row]>
__global__ void moe_combine_bwd_kernel(const uint4* __restrict__ dy, const uint4* __restrict__ yg,
                                       const int32_t* __restrict__ slot_of_row,
                                       const int32_t* __restrict__ offsets_padded, const float* __restrict__ sel_w,
                                       uint4* __restrict__ dyg, float* __restrict__ dw, int E, int k, int H8,
                                       int64_t max_rows, float alpha) {
    const int64_t row = (int64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (row >= max_rows || row >= offsets_padded[E]) return;
    const int slot = slot_of_row[row];
    uint4* dst = dyg + row * H8;
    if (slot < 0) {
        for (int i = lane; i < H8; i += 32) dst[i] = make_uint4(0, 0, 0, 0);
        return;
    }
    const float w = bf16_round(sel_w[slot]) * alpha;
    const uint4* g = dy + int64_t(slot / k) * H8;
    const uint4* y = yg + row * H8;
    float dot = 0.f;
    for (int i = lane; i < H8; i += 32) {
        float a[8], b[8], o[8];
        unpack8(__ldg(g + i), a);
        unpack8(__ldg(y + i), b);
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            dot += a[q] * b[q];
            o[q] = a[q] * w;
        }
        dst[i] = pack8(o);
    }
    dot = warp_sum(dot);
    if (lane == 0) dw[slot] = dot * alpha;
}

// dx[t] = sum_j dX_g[row_of_slot[t*k+j]]   (one warp per token)
__global__ void moe_token_sum_kernel(const uint4* __restrict__ dxg, const int32_t* __restrict__ row_of_slot,
                                     uint4* __restrict__ dx, int64_t T, int k, int H8) {
    const int64_t t = (int64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (t >= T) return;
    for (int i = lane; i < H8; i += 32) {
        float acc[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[q] = 0.f;
        for (int j = 0; j < k; ++j) {
            float f[8];
            unpack8(__ldg(dxg + int64_t(row_of_slot[t * k + j]) * H8 + i), f);
#pragma unroll
            for (int q = 0; q < 8; ++q) acc[q] += f[q];
        }
        dx[t * H8 + i] = pack8(acc);
    }
}

// softmax-over-selected backward -> dense dlogits bf16 [T, E] (zeros for unselected experts); one thread per token
__global__ void moe_router_bwd_kernel(const int32_t* __restrict__ sel_idx, const float* __restrict__ sel_w,
                                      const float* __restrict__ dw, __nv_bfloat16* __restrict__ dlogits, int64_t T,
                                      int E, int k) {
    const int64_t t = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (t >= T) return;
    for (int e = 0; e < E; ++e) dlogits[t * E + e] = __float2bfloat16_rn(0.f);
    float dot = 0.f;
    for (int j = 0; j < k; ++j) dot += sel_w[t * k + j] * dw[t * k + j];
    for (int j = 0; j < k; ++j) {
        const float w = sel_w[t * k + j];
        dlogits[t * E + sel_idx[t * k + j]] = __float2bfloat16_rn(w * (dw[t * k + j] - dot));
    }
}

inline int64_t align256(int64_t x) { return (x + 255) & ~int64_t(255); }

}  // namespace

extern "C" int64_t dolomite_b200_moe_max_rows(int64_t T, int E, int k) { return (T * k + int64_t(E) * (MOE_PAD - 1)) / MOE_PAD * MOE_PAD + MOE_PAD; }

extern "C" int dolomite_b200_moe_route(const void* router_logits, int64_t T, int E, int k, int32_t* sel_idx,
                                       float* sel_w, int32_t* counts, int32_t* offsets_padded, int32_t* m_tile_group,
                                       int32_t* cursors, int32_t* row_of_slot, int32_t* slot_of_row,
                                       int32_t* token_of_row, void* stream) {
    DOLO_REQUIRE(E > 0 && E <= 256, "moe_route: num_experts=%d must be in [1, 256]", E);
    DOLO_REQUIRE(k > 0 && k <= 8 && k <= E, "moe_route: top-k=%d must be in [1, min(8, E)]", k);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int64_t max_rows = dolomite_b200_moe_max_rows(T, E, k);
    const int max_tiles = int(max_rows / MOE_TILE);
    DOLO_CUDA_OK(cudaMemsetAsync(counts, 0, sizeof(int32_t) * E, st));
    DOLO_CUDA_OK(cudaMemsetAsync(slot_of_row, 0xFF, sizeof(int32_t) * max_rows, st));
    DOLO_CUDA_OK(cudaMemsetAsync(token_of_row, 0, sizeof(int32_t) * max_rows, st));  // padding rows read token 0 (never used)
    if (T > 0) {
        const int64_t blocks = (T * 32 + 255) / 256;
        moe_route_kernel<<<(unsigned)blocks, 256, 0, st>>>(static_cast<const __nv_bfloat16*>(router_logits), T, E, k,
                                                           sel_idx, sel_w, counts);
        DOLO_LAUNCH_OK("moe_route");
    }
    moe_plan_kernel<<<1, 256, 0, st>>>(counts, E, offsets_padded, m_tile_group, max_tiles, cursors);
    DOLO_LAUNCH_OK("moe_plan");
    if (T > 0) {
        const int64_t n = T * k;
        moe_assign_kernel<<<E, 1024, 0, st>>>(sel_idx, n, offsets_padded, row_of_slot, slot_of_row, token_of_row, k);
        DOLO_LAUNCH_OK("moe_assign");
    }
    return DOLO_OK;
}

extern "C" int dolomite_b200_moe_gather(const void* x, void* xg, const int32_t* slot_of_row,
                                        const int32_t* offsets_padded, int64_t T, int E, int k, int H, void* stream) {
    DOLO_REQUIRE(H % 8 == 0, "moe_gather: H %% 8");
    const int64_t max_rows = dolomite_b200_moe_max_rows(T, E, k);
    const int64_t blocks = (max_rows * 32 + 255) / 256;
    moe_gather_kernel<<<(unsigned)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const uint4*>(x), static_cast<uint4*>(xg), slot_of_row, offsets_padded, E, k, H / 8, max_rows);
    DOLO_LAUNCH_OK("moe_gather");
    return DOLO_OK;
}

extern "C" int dolomite_b200_moe_combine(const void* yg, const int32_t* row_of_slot, const float* sel_w, const void* c,
                                         void* out, int64_t T, int k, int H, float alpha, void* stream) {
    DOLO_REQUIRE(H % 8 == 0, "moe_combine: H %% 8");
    if (T == 0) return DOLO_OK;
    const int64_t blocks = (T * 32 + 255) / 256;
    moe_combine_kernel<<<(unsigned)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const uint4*>(yg), row_of_slot, sel_w, static_cast<const uint4*>(c), static_cast<uint4*>(out), T, k,
        H / 8, alpha);
    DOLO_LAUNCH_OK("moe_combine");
    return DOLO_OK;
}

extern "C" int dolomite_b200_moe_combine_bwd(const void* dy, const void* yg, const int32_t* slot_of_row,
                                             const int32_t* offsets_padded, const float* sel_w, void* dyg, float* dw,
                                             int64_t T, int E, int k, int H, float alpha, void* stream) {
    DOLO_REQUIRE(H % 8 == 0, "moe_combine_bwd: H %% 8");
    const int64_t max_rows = dolomite_b200_moe_max_rows(T, E, k);
    const int64_t blocks = (max_rows * 32 + 255) / 256;
    moe_combine_bwd_kernel<<<(unsigned)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const uint4*>(dy), static_cast<const uint4*>(yg), slot_of_row, offsets_padded, sel_w,
        static_cast<uint4*>(dyg), dw, E, k, H / 8, max_rows, alpha);
    DOLO_LAUNCH_OK("moe_combine_bwd");
    return DOLO_OK;
}

extern "C" int dolomite_b200_moe_token_sum(const void* dxg, const int32_t* row_of_slot, void* dx, int64_t T, int k,
                                           int H, void* stream) {
    DOLO_REQUIRE(H % 8 == 0, "moe_token_sum: H %% 8");
    if (T == 0) return DOLO_OK;
    const int64_t blocks = (T * 32 + 255) / 256;
    moe_token_sum_kernel<<<(unsigned)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const uint4*>(dxg), row_of_slot, static_cast<uint4*>(dx), T, k, H / 8);
    DOLO_LAUNCH_OK("moe_token_sum");
    return DOLO_OK;
}

extern "C" int dolomite_b200_moe_router_bwd(const int32_t* sel_idx, const float* sel_w, const float* dw, void* dlogits,
                                            int64_t T, int E, int k, void* stream) {
    if (T == 0) return DOLO_OK;
    moe_router_bwd_kernel<<<(unsigned)((T + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        sel_idx, sel_w, dw, static_cast<__nv_bfloat16*>(dlogits), T, E, k);
    DOLO_LAUNCH_OK("moe_router_bwd");
    return DOLO_OK;
}
