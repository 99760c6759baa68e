// Packed attention of new tokens against a KV cache (reference: attention/sdpa.py:11-83 and attention/flash.py:16-140 with
// `past_key_values` and a query block of several tokens; causal mask from past_length on, gpt_dolomite/base.py:300-349).
//
// Sequence b has past[b] cached tokens and n[b] = cu_new[b + 1] - cu_new[b] >= 0 new ones, whose keys / values the caller
// has already written at cache positions past[b] .. past[b] + n[b] - 1.  New token i attends to cache keys 0 .. past[b] + i.
// n[b] == 0: nothing is computed or written for the sequence.
//
// One CTA = one consumer warpgroup of 64 M rows of one kv group of one sequence.  Row f of the sequence is the pair (new token
// f / g, q head f % g of the group), g = q_per_group, so one CTA reads each K / V tile once for all the q heads of its
// group: with few new tokens (a handful per sequence, or MQA) the 64 rows are still filled.  Thread 0 streams 64-key K / V
// tiles from cache position 0 in order through a 2-stage TMA ring; per tile
//     S = Q K_j^T (SS, 64 x 64 fp32)   online softmax   O += P V_j (RS)
// as attn_wide_fwd_kernel, whose register (o 128 + S 32 + P 16 at head_dim 256) and shared-memory budget one kernel body
// follows for every head dim.  The rows of a tile belong to different tokens, so Q is gathered by the threads into the
// swizzled chunk layout a TMA box would produce.  A key tile every row of the CTA fully masks changes no row: the result of a
// query row does not depend on how the new tokens of a sequence are split across calls.
//
// Cache layout: k_cache / v_cache [B, L_max, n_groups * head_dim] bf16 (attention_decode.cu).  Positions >= past + n of
// the last key tile (the next sequence's cache, or stale values) are masked, and their V rows are zeroed in shared memory so
// that 0 * NaN never reaches the accumulators.
// ALIBI: the logit of cache key k of head h gets attn_alibi_bias(slope_h, k), as attn_decode.
#include "attention_common.cuh"
#include "../../include/dolomite_b200.h"

using namespace dolo;

namespace {

constexpr int CACHE_M = 64;        // M rows (token, q head) per CTA
constexpr int CACHE_KT = 64;       // keys per K / V tile
constexpr int CACHE_STAGES = 2;    // depth of the K / V ring
constexpr int CACHE_THREADS = 128;

struct CacheParams {
    const __nv_bfloat16* qkv;
    int64_t row_stride;
    const int32_t* cu_new;      // [B + 1]
    const int32_t* past;        // [B]
    __nv_bfloat16* out;         // [sum n, n_heads * HD]
    int64_t L_max;
    int n_groups, q_per_group, n_heads;
    float scale_log2;
    const float* alibi_slopes;  // [n_heads] fp32, read by the ALIBI instances only
};

template <int HD, bool ALIBI>
__global__ void __launch_bounds__(CACHE_THREADS, 1)
    attn_cache_kernel(const __grid_constant__ CUtensorMap tk64, const __grid_constant__ CUtensorMap tkR,
                      const __grid_constant__ CUtensorMap tv64, const __grid_constant__ CUtensorMap tvR, const CacheParams p) {
    using CH = HeadChunks<HD>;
    constexpr int T_BYTES = CH::tile_bytes(CACHE_KT);
    static_assert(CH::tile_bytes(CACHE_M) == T_BYTES, "Q and K / V tiles have the same shape");

    const int b = blockIdx.z, group = blockIdx.y, m0 = blockIdx.x * CACHE_M;
    const int g = p.q_per_group;
    const int tok0 = p.cu_new[b];
    const int n = p.cu_new[b + 1] - tok0;
    const int rows = n * g;
    if (m0 >= rows) return;  // uniform for the whole CTA
    const int past = p.past[b];
    const int end = past + n;  // cache positions of the call: keys 0 .. end - 1
    const int n_kt = (end + CACHE_KT - 1) / CACHE_KT;
    const int kv_row0 = b * int(p.L_max);  // B * L_max < 2^31 (host check)

    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_align_1024(smem_raw);
    uint8_t* sQ = smem;
    uint8_t* sK = sQ + T_BYTES;                  // [CACHE_STAGES]
    uint8_t* sV = sK + CACHE_STAGES * T_BYTES;   // [CACHE_STAGES]
    uint64_t* bars = reinterpret_cast<uint64_t*>(sV + CACHE_STAGES * T_BYTES);
    uint64_t* kv_full = bars;                    // [CACHE_STAGES]
    uint64_t* kv_empty = bars + CACHE_STAGES;    // [CACHE_STAGES], one arrive per warp

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    auto load_kv = [&](int j, int s) {
        mbar_expect_tx(&kv_full[s], 2 * T_BYTES);
        tma_load_chunked<HD, CACHE_KT>(sK + s * T_BYTES, &tk64, &tkR, &kv_full[s], group * HD, kv_row0 + j * CACHE_KT);
        tma_load_chunked<HD, CACHE_KT>(sV + s * T_BYTES, &tv64, &tvR, &kv_full[s], group * HD, kv_row0 + j * CACHE_KT);
    };
    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tk64);
        tma_prefetch_desc(&tv64);
        if (CH::REM > 0) {
            tma_prefetch_desc(&tkR);
            tma_prefetch_desc(&tvR);
        }
        for (int i = 0; i < CACHE_STAGES; ++i) {
            mbar_init(&kv_full[i], 1);
            mbar_init(&kv_empty[i], CACHE_THREADS / 32);
        }
        mbar_fence_init();
        for (int j = 0; j < CACHE_STAGES && j < n_kt; ++j) load_kv(j, j);
    }

    // ---------------- Q: gather the 64 (token, head) rows into the swizzled chunk layout ----------------
    // 16-byte unit u of row r of a chunk of w columns sits at unit u ^ swz(r) of the row: the SWIZZLE_128B / 64B / 32B
    // patterns of the TMA unit (byte address bits [4, 7) ^= bits [7, 10) / [4, 6) ^= [7, 9) / bit 4 ^= bit 7)
    constexpr int UNITS = HD / 8;
    for (int e = threadIdx.x; e < CACHE_M * UNITS; e += CACHE_THREADS) {
        const int r = e / UNITS, u = e - (e / UNITS) * UNITS;
        const int f = m0 + r;
        uint4 val = make_uint4(0u, 0u, 0u, 0u);
        if (f < rows) {
            const int i = f / g, slot = f - (f / g) * g;
            val = *reinterpret_cast<const uint4*>(p.qkv + int64_t(tok0 + i) * p.row_stride +
                                                  int64_t(group * (g + 2) + slot) * HD + u * 8);
        }
        const int c = u >> 3, uc = u & 7;
        const int w = CH::width(c);
        const int swz = w == 64 ? (r & 7) : (w == 32 ? ((r >> 1) & 3) : ((r >> 2) & 1));
        *reinterpret_cast<uint4*>(sQ + CH::offset(c, CACHE_M) + r * 2 * w + ((uc ^ swz) << 4)) = val;
    }
    fence_proxy_async_smem();  // generic-proxy writes of Q, read by wgmma
    __syncthreads();

    const int wr = (warp & 3) * 16 + (lane >> 2);  // first of the two accumulator rows of this thread (and wr + 8)
    const int wc = 2 * (lane & 3);                 // first accumulator column inside each n8 block
    int lim[2];                                     // last key of each row
    float slope[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int f = min(m0 + wr + 8 * h, rows - 1);  // a row past the new tokens is computed as the last one, not written
        lim[h] = past + f / g;
        slope[h] = ALIBI ? __ldg(p.alibi_slopes + group * g + (m0 + wr + 8 * h) % g) : 0.f;
    }
    const int j_mask = (past + m0 / g) / CACHE_KT;  // first key tile with a key past some row's last key
    const uint32_t sq = smem_u32(sQ);

    float o[HD / 2];
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
    // row max (raw score; ALIBI: log2 units of the biased logit), thread-partial row sum
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};

    for (int j = 0; j < n_kt; ++j) {
        const int s = j & (CACHE_STAGES - 1);
        mbar_wait(&kv_full[s], (j / CACHE_STAGES) & 1, 71);
        const int r_end = end - j * CACHE_KT;  // rows >= r_end of this tile are past the keys of the call
        if (r_end < CACHE_KT) {                 // last tile, CTA-uniform
            for (int e = threadIdx.x; e < (CACHE_KT - r_end) * (HD / 8); e += CACHE_THREADS) {
                const int r = r_end + e / (HD / 8), u = e % (HD / 8);
                const int c = u >> 3, w = CH::width(c);
                *reinterpret_cast<uint4*>(sV + s * T_BYTES + CH::offset(c, CACHE_KT) + r * 2 * w + ((u & 7) << 4)) =
                    make_uint4(0u, 0u, 0u, 0u);  // whole rows: the swizzle permutes units inside a row only
            }
            fence_proxy_async_smem();
            __syncthreads();
        }
        const uint32_t sk = smem_u32(sK + s * T_BYTES), sv = smem_u32(sV + s * T_BYTES);
        float sc[CACHE_KT / 2];
        wgmma_fence();
#pragma unroll
        for (int c = 0; c < CH::NCHUNK; ++c) {
            const int w = CH::width(c);
#pragma unroll
            for (int k = 0; k < w / 16; ++k)
                wgmma_ss<CACHE_KT, 0, 0>(sc, chunk_desc_kmajor(sq + CH::offset(c, CACHE_M), w, k),
                                         chunk_desc_kmajor(sk + CH::offset(c, CACHE_KT), w, k), (c != 0 || k != 0) ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        reg_fence<CACHE_KT / 2>(sc);

        // ---------------- online softmax over this key tile ----------------
        const bool mask = j >= j_mask;
        const int kbase = j * CACHE_KT + wc;
        if constexpr (ALIBI) {  // sc <- log2(e) * (scale * s + bias_k)
#pragma unroll
            for (int bb = 0; bb < CACHE_KT / 8; ++bb)
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int e = 0; e < 2; ++e)
                        sc[4 * bb + 2 * h + e] = fmaf(sc[4 * bb + 2 * h + e], p.scale_log2,
                                                      attn_alibi_bias(slope[h], kbase + 8 * bb + e) * ATT_LOG2E);
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            float mx = m_run[h];
#pragma unroll
            for (int bb = 0; bb < CACHE_KT / 8; ++bb)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    float& x = sc[4 * bb + 2 * h + e];
                    if (mask && kbase + 8 * bb + e > lim[h]) x = -INFINITY;
                    mx = fmaxf(mx, x);
                }
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            // key 0 precedes every query: the row max is finite from key tile 0 on
            const float corr = ALIBI ? fast_exp2(m_run[h] - mx) : fast_exp2((m_run[h] - mx) * p.scale_log2);
            const float neg_m = ALIBI ? -mx : -mx * p.scale_log2;
            float lsum = 0.f;
#pragma unroll
            for (int bb = 0; bb < CACHE_KT / 8; ++bb)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    float& x = sc[4 * bb + 2 * h + e];
                    const float pr = ALIBI ? fast_exp2(x + neg_m) : fast_exp2(fmaf(x, p.scale_log2, neg_m));
                    lsum += pr;
                    x = pr;
                }
            l_run[h] = l_run[h] * corr + lsum;
            m_run[h] = mx;
#pragma unroll
            for (int bb = 0; bb < HD / 8; ++bb) {
                o[4 * bb + 2 * h] *= corr;
                o[4 * bb + 2 * h + 1] *= corr;
            }
        }
        uint32_t pa[CACHE_KT / 16][4];
#pragma unroll
        for (int kk = 0; kk < CACHE_KT / 16; ++kk) acc_to_a_frag(sc, kk, pa[kk]);

        // ---------------- O += P V_j ----------------
        wgmma_fence();
#pragma unroll
        for (int c = 0; c < CH::NCHUNK; ++c) {
#pragma unroll
            for (int kk = 0; kk < CACHE_KT / 16; ++kk) {
                if (CH::width(c) == 64)
                    wgmma_rs<64, 1>(o + CH::col(c) / 2, pa[kk], chunk_desc_mnmajor(sv + CH::offset(c, CACHE_KT), 64, kk), 1u);
                else
                    wgmma_rs<(CH::REM ? CH::REM : 16), 1>(o + CH::col(c) / 2, pa[kk],
                                                          chunk_desc_mnmajor(sv + CH::offset(c, CACHE_KT), CH::REM, kk), 1u);
            }
        }
        wgmma_commit();
        wgmma_wait<0>();
        reg_fence<HD / 2>(o);

        if (lane == 0) mbar_arrive(&kv_empty[s]);
        if (threadIdx.x == 0 && j + CACHE_STAGES < n_kt) {
            mbar_wait(&kv_empty[s], (j / CACHE_STAGES) & 1, 72);  // every warp is done with tile j
            load_kv(j + CACHE_STAGES, s);
        }
        __syncwarp();
    }

    // ---------------- epilogue: O / l ----------------
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        float l = l_run[h];
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        const int f = m0 + wr + 8 * h;
        if (f >= rows) continue;
        const int i = f / g, slot = f - (f / g) * g;
        const float inv_l = l > 0.f ? 1.f / l : 0.f;
        __nv_bfloat16* orow = p.out + int64_t(tok0 + i) * (int64_t(p.n_heads) * HD) + int64_t(group * g + slot) * HD + wc;
#pragma unroll
        for (int bb = 0; bb < HD / 8; ++bb)
            *reinterpret_cast<uint32_t*>(orow + 8 * bb) = pack_bf16(o[4 * bb + 2 * h] * inv_l, o[4 * bb + 2 * h + 1] * inv_l);
    }
}

template <int HD, bool ALIBI>
int launch_cache(const CacheParams& p, const void* k_cache, const void* v_cache, int batch, int max_new, cudaStream_t st) {
    using CH = HeadChunks<HD>;
    CUtensorMap k64, kR, v64, vR;
    const int64_t ld = int64_t(p.n_groups) * HD, rows = int64_t(batch) * p.L_max;
    int rc = attn_make_maps<HD>(k_cache, ld, rows, &k64, &kR);
    if (rc) return rc;
    rc = attn_make_maps<HD>(v_cache, ld, rows, &v64, &vR);
    if (rc) return rc;
    constexpr int smem_bytes = 1024 + (1 + 2 * CACHE_STAGES) * CH::tile_bytes(CACHE_KT) + 128;
    static_assert(smem_bytes <= 232448, "KV-cache attention shared memory budget exceeded");
    auto kern = attn_cache_kernel<HD, ALIBI>;
    static bool attr_set = false;
    if (!attr_set) {
        DOLO_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
        attr_set = true;
    }
    const int64_t m_tiles = (int64_t(max_new) * p.q_per_group + CACHE_M - 1) / CACHE_M;
    dim3 grid(unsigned(m_tiles), unsigned(p.n_groups), unsigned(batch));
    kern<<<grid, CACHE_THREADS, smem_bytes, st>>>(k64, kR, v64, vR, p);
    DOLO_LAUNCH_OK("attn_cache");
    return DOLO_OK;
}

template <int HD>
int launch_cache_any(const CacheParams& p, const void* k_cache, const void* v_cache, int batch, int max_new, cudaStream_t st) {
    if (p.alibi_slopes != nullptr) return launch_cache<HD, true>(p, k_cache, v_cache, batch, max_new, st);
    return launch_cache<HD, false>(p, k_cache, v_cache, batch, max_new, st);
}

// alibi_slopes == nullptr: the plain kernel
int attn_cache(const void* qkv, int64_t row_stride, const int32_t* cu_new, const int32_t* past, const void* k_cache,
               const void* v_cache, void* out, int batch, int max_new, int max_end, int64_t L_max, int n_groups,
               int q_per_group, int head_dim, float softmax_scale, const float* alibi_slopes, void* stream) {
    DOLO_REQUIRE(batch >= 0 && max_new >= 0 && L_max > 0, "attn_cache: bad sizes");
    DOLO_REQUIRE(max_new <= max_end && max_end <= L_max, "attn_cache: past + n (up to %d) exceeds the cache length %lld",
                 max_end, (long long)L_max);
    if (batch == 0 || max_new == 0) return DOLO_OK;
    DOLO_REQUIRE(n_groups > 0 && q_per_group > 0, "attn_cache: bad head grouping");
    DOLO_REQUIRE(batch <= 65535 && n_groups <= 65535 && int64_t(batch) * L_max < (1ll << 31) &&
                     int64_t(max_new) * q_per_group < (1ll << 31),
                 "attn_cache: grid too large");
    switch (head_dim) {
        case 16: case 32: case 64: case 80: case 96: case 128: case 160: case 192: case 256: break;
        default: return dolo_set_error("attn_cache: unsupported head_dim %d (supported: 16,32,64,80,96,128,160,192,256)", head_dim);
    }
    DOLO_REQUIRE(row_stride % 8 == 0 && (reinterpret_cast<uintptr_t>(qkv) & 15) == 0 &&
                     (reinterpret_cast<uintptr_t>(k_cache) & 15) == 0 && (reinterpret_cast<uintptr_t>(v_cache) & 15) == 0 &&
                     (reinterpret_cast<uintptr_t>(out) & 15) == 0,
                 "attn_cache: alignment");
    CacheParams p{};
    p.qkv = static_cast<const __nv_bfloat16*>(qkv);
    p.row_stride = row_stride;
    p.cu_new = cu_new;
    p.past = past;
    p.out = static_cast<__nv_bfloat16*>(out);
    p.L_max = L_max;
    p.n_groups = n_groups;
    p.q_per_group = q_per_group;
    p.n_heads = n_groups * q_per_group;
    p.scale_log2 = softmax_scale * 1.4426950408889634f;
    p.alibi_slopes = alibi_slopes;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    switch (head_dim) {
        case 16: return launch_cache_any<16>(p, k_cache, v_cache, batch, max_new, st);
        case 32: return launch_cache_any<32>(p, k_cache, v_cache, batch, max_new, st);
        case 64: return launch_cache_any<64>(p, k_cache, v_cache, batch, max_new, st);
        case 80: return launch_cache_any<80>(p, k_cache, v_cache, batch, max_new, st);
        case 96: return launch_cache_any<96>(p, k_cache, v_cache, batch, max_new, st);
        case 128: return launch_cache_any<128>(p, k_cache, v_cache, batch, max_new, st);
        case 160: return launch_cache_any<160>(p, k_cache, v_cache, batch, max_new, st);
        case 192: return launch_cache_any<192>(p, k_cache, v_cache, batch, max_new, st);
        default: return launch_cache_any<256>(p, k_cache, v_cache, batch, max_new, st);
    }
}

}  // namespace

extern "C" int dolomite_b200_attn_cache(const void* qkv, int64_t row_stride, const int32_t* cu_new, const int32_t* past,
                                        const void* k_cache, const void* v_cache, void* out, int batch, int max_new,
                                        int max_end, int64_t L_max, int n_groups, int q_per_group, int head_dim,
                                        float softmax_scale, void* stream) {
    return attn_cache(qkv, row_stride, cu_new, past, k_cache, v_cache, out, batch, max_new, max_end, L_max, n_groups,
                      q_per_group, head_dim, softmax_scale, nullptr, stream);
}

extern "C" int dolomite_b200_attn_cache_alibi(const void* qkv, int64_t row_stride, const int32_t* cu_new,
                                              const int32_t* past, const void* k_cache, const void* v_cache, void* out,
                                              int batch, int max_new, int max_end, int64_t L_max, int n_groups,
                                              int q_per_group, int head_dim, float softmax_scale,
                                              const float* alibi_slopes, void* stream) {
    DOLO_REQUIRE(alibi_slopes != nullptr, "attn_cache_alibi: alibi_slopes is null");
    return attn_cache(qkv, row_stride, cu_new, past, k_cache, v_cache, out, batch, max_new, max_end, L_max, n_groups,
                      q_per_group, head_dim, softmax_scale, alibi_slopes, stream);
}
