// Packed var-len causal attention forward on wgmma (replaces flash_attn_varlen_func at
// attention/padding_free.py:51-62).
//
// One CTA = one 128-row query tile of one head of one document, two warpgroups of 64 query rows each.  Thread 0 also
// issues the TMA loads: the Q tile once, then (K_j, V_j) tiles through a 2-stage ring.  Per key tile every warpgroup runs
//     S = Q K_j^T        (wgmma SS, fp32 scores in registers, 64 x 128 per warpgroup)
//     online softmax     (each thread holds two query rows x 32 keys; row max / sum over the quad of a row)
//     O += P V_j         (wgmma RS: P as the bf16 register A operand, V MN-major from shared memory)
// and finally writes O / l and the natural-log LSE.
// ALIBI: the logits are scale * s + bias_k with a per-(head, key) bias (see attn_alibi_bias); the running row max is then
// kept in log2 units of the biased logit instead of in raw-score units.
#include "attention_common.cuh"
#include "../../include/dolomite_b200.h"

using namespace dolo;

namespace {

constexpr int FWD_THREADS = 256;
constexpr int KV_STAGES = 2;

struct FwdParams {
    __nv_bfloat16* out;
    float* lse;
    const int32_t* cu_seqlens;
    int n_docs;
    int64_t T;
    int n_groups, q_per_group;
    int n_heads;
    float scale_log2;  // softmax_scale * log2(e)
    float scale;
    AttnDropout drop;  // threshold 0: none
    int head_chunk;    // CTA order (attention_common.cuh: attn_cta_order): heads per chunk, 0 = tiles fastest
    int n_tile_slots;  // upper bound of the number of query tiles (the grid has n_tile_slots x n_heads CTAs)
    const float* alibi_slopes;  // [n_heads] fp32, read by the ALIBI instances only
};

template <int HD, bool ALIBI>
__global__ void __launch_bounds__(FWD_THREADS, 1)
    attn_fwd_kernel(const __grid_constant__ CUtensorMap tmap64, const __grid_constant__ CUtensorMap tmapR,
                    const FwdParams p) {
    using CH = HeadChunks<HD>;
    constexpr int TILE_BYTES = CH::tile_bytes(ATT_TILE);

    int ti, head;
    attn_cta_order(p.head_chunk, p.n_tile_slots, ti, head);
    ti = p.n_tile_slots - 1 - ti;  // long (late) tiles first
    const TileLoc loc = locate_tile(p.cu_seqlens, p.n_docs, ti);
    if (!loc.valid) return;  // uniform for the whole CTA
    const int group = head / p.q_per_group, slot = head % p.q_per_group;
    const int q_col = (group * (p.q_per_group + 2) + slot) * HD;
    const int k_col = (group * (p.q_per_group + 2) + p.q_per_group) * HD;
    const int v_col = k_col + HD;
    const int q0 = loc.tile * ATT_TILE;  // first query (doc-relative) of this tile
    const int n_kv = loc.tile + 1;       // causal: key tiles 0 .. tile

    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_align_1024(smem_raw);
    uint8_t* sQ = smem;
    uint8_t* sK = sQ + TILE_BYTES;              // [KV_STAGES]
    uint8_t* sV = sK + KV_STAGES * TILE_BYTES;  // [KV_STAGES]
    uint64_t* bars = reinterpret_cast<uint64_t*>(sV + KV_STAGES * TILE_BYTES);
    uint64_t* q_full = bars;        // 1
    uint64_t* kv_full = bars + 1;   // [KV_STAGES]
    uint64_t* kv_empty = bars + 3;  // [KV_STAGES], one arrive per warp

    const int wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    auto load_kv = [&](int j, int s) {
        mbar_expect_tx(&kv_full[s], 2 * TILE_BYTES);
        tma_load_chunked<HD, ATT_TILE>(sK + s * TILE_BYTES, &tmap64, &tmapR, &kv_full[s], k_col, loc.doc_start + j * ATT_TILE);
        tma_load_chunked<HD, ATT_TILE>(sV + s * TILE_BYTES, &tmap64, &tmapR, &kv_full[s], v_col, loc.doc_start + j * ATT_TILE);
    };
    if (threadIdx.x == 0) {
        if (CH::NC64 > 0) tma_prefetch_desc(&tmap64);
        if (CH::REM > 0) tma_prefetch_desc(&tmapR);
        mbar_init(q_full, 1);
        for (int i = 0; i < KV_STAGES; ++i) {
            mbar_init(&kv_full[i], 1);
            mbar_init(&kv_empty[i], FWD_THREADS / 32);
        }
        mbar_fence_init();
        mbar_expect_tx(q_full, TILE_BYTES);
        tma_load_chunked<HD, ATT_TILE>(sQ, &tmap64, &tmapR, q_full, q_col, loc.doc_start + q0);
        for (int j = 0; j < KV_STAGES && j < n_kv; ++j) load_kv(j, j);
    }
    __syncthreads();

    const int wr = (warp & 3) * 16 + (lane >> 2);  // first of the two accumulator rows of this thread (and wr + 8)
    const int wc = 2 * (lane & 3);                 // first accumulator column inside each n8 block
    const int qr[2] = {q0 + wg * 64 + wr, q0 + wg * 64 + wr + 8};  // doc-relative queries of the two rows
    const bool drop = p.drop.threshold != 0;
    const uint32_t head_key = dropout_head_key(uint32_t(head), p.drop.key0, p.drop.key1);
    const uint32_t sq = smem_u32(sQ);

    float o[HD / 2];
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
    // row max (raw score; ALIBI: log2 units of the biased logit), thread-partial row sum
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    const float slope = ALIBI ? __ldg(p.alibi_slopes + head) : 0.f;

    mbar_wait(q_full, 0, 10);
    for (int j = 0; j < n_kv; ++j) {
        const int s = j & (KV_STAGES - 1);
        mbar_wait(&kv_full[s], (j / KV_STAGES) & 1, 11);
        const uint32_t sk = smem_u32(sK + s * TILE_BYTES), sv = smem_u32(sV + s * TILE_BYTES);
        float sc[ATT_TILE / 2];
        wgmma_fence();
#pragma unroll
        for (int c = 0; c < CH::NCHUNK; ++c) {
            const int w = CH::width(c);
#pragma unroll
            for (int k = 0; k < w / 16; ++k)
                wgmma_ss<ATT_TILE, 0, 0>(sc, chunk_desc_kmajor(sq + CH::offset(c, ATT_TILE) + wg * 64 * 2 * w, w, k),
                                         chunk_desc_kmajor(sk + CH::offset(c, ATT_TILE), w, k), (c != 0 || k != 0) ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        reg_fence<ATT_TILE / 2>(sc);

        // ---------------- online softmax over this key tile ----------------
        const bool diag = j == loc.tile;  // only the diagonal tile has keys past a query of the tile
        const int kbase = j * ATT_TILE + wc;
        if constexpr (ALIBI) {  // sc <- log2(e) * (scale * s + bias_k): one bias per key column, shared by both rows
#pragma unroll
            for (int b = 0; b < ATT_TILE / 8; ++b)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const float bl = attn_alibi_bias(slope, kbase + 8 * b + e) * ATT_LOG2E;
                    sc[4 * b + e] = fmaf(sc[4 * b + e], p.scale_log2, bl);
                    sc[4 * b + 2 + e] = fmaf(sc[4 * b + 2 + e], p.scale_log2, bl);
                }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            float mx = m_run[h];
#pragma unroll
            for (int b = 0; b < ATT_TILE / 8; ++b)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    float& x = sc[4 * b + 2 * h + e];
                    if (diag && kbase + 8 * b + e > qr[h]) x = -INFINITY;
                    mx = fmaxf(mx, x);
                }
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            // key 0 of every tile j <= tile precedes every query of the tile: the row max is finite from tile 0 on
            const float corr = ALIBI ? fast_exp2(m_run[h] - mx) : fast_exp2((m_run[h] - mx) * p.scale_log2);
            const float neg_m = ALIBI ? -mx : -mx * p.scale_log2;
            float lsum = 0.f;
#pragma unroll
            for (int b = 0; b < ATT_TILE / 8; ++b)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    float& x = sc[4 * b + 2 * h + e];
                    // exp2(-inf) = 0 for masked keys
                    float pr = ALIBI ? fast_exp2(x + neg_m) : fast_exp2(fmaf(x, p.scale_log2, neg_m));
                    lsum += pr;
                    if (drop)  // the row sum above is that of the undropped probabilities
                        pr *= attn_drop_scale(p.drop, head_key, loc.doc_start + qr[h], loc.doc_start + kbase + 8 * b + e);
                    x = pr;
                }
            l_run[h] = l_run[h] * corr + lsum;
            m_run[h] = mx;
#pragma unroll
            for (int b = 0; b < HD / 8; ++b) {
                o[4 * b + 2 * h] *= corr;
                o[4 * b + 2 * h + 1] *= corr;
            }
        }
        uint32_t pa[ATT_TILE / 16][4];
#pragma unroll
        for (int kk = 0; kk < ATT_TILE / 16; ++kk) acc_to_a_frag(sc, kk, pa[kk]);

        // ---------------- O += P V_j ----------------
        wgmma_fence();
#pragma unroll
        for (int c = 0; c < CH::NCHUNK; ++c) {
#pragma unroll
            for (int kk = 0; kk < ATT_TILE / 16; ++kk) {
                if (CH::width(c) == 64)
                    wgmma_rs<64, 1>(o + CH::col(c) / 2, pa[kk], chunk_desc_mnmajor(sv + CH::offset(c, ATT_TILE), 64, kk), 1u);
                else
                    wgmma_rs<(CH::REM ? CH::REM : 16), 1>(o + CH::col(c) / 2, pa[kk],
                                                          chunk_desc_mnmajor(sv + CH::offset(c, ATT_TILE), CH::REM, kk), 1u);
            }
        }
        wgmma_commit();
        wgmma_wait<0>();
        reg_fence<HD / 2>(o);
        if (lane == 0) mbar_arrive(&kv_empty[s]);
        if (threadIdx.x == 0 && j + KV_STAGES < n_kv) {
            mbar_wait(&kv_empty[s], (j / KV_STAGES) & 1, 12);  // both warpgroups are done with tile j
            load_kv(j + KV_STAGES, s);
        }
        __syncwarp();
    }

    // ---------------- epilogue: O / l, LSE ----------------
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        float l = l_run[h];
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        if (qr[h] >= loc.doc_len) continue;
        const float inv_l = l > 0.f ? 1.f / l : 0.f;
        const int64_t row = loc.doc_start + qr[h];
        __nv_bfloat16* orow = p.out + row * (int64_t(p.n_heads) * HD) + int64_t(head) * HD + wc;
#pragma unroll
        for (int b = 0; b < HD / 8; ++b)
            *reinterpret_cast<uint32_t*>(orow + 8 * b) = pack_bf16(o[4 * b + 2 * h] * inv_l, o[4 * b + 2 * h + 1] * inv_l);
        if ((lane & 3) == 0)
            p.lse[int64_t(head) * p.T + row] = (ALIBI ? m_run[h] * ATT_LN2 : m_run[h] * p.scale) + logf(l);
    }
}

template <int HD, bool ALIBI>
int launch_fwd(const void* qkv, int64_t row_stride, const FwdParams& p, cudaStream_t st) {
    using CH = HeadChunks<HD>;
    CUtensorMap t64, tR;
    int rc = attn_make_maps<HD>(qkv, row_stride, p.T, &t64, &tR);
    if (rc) return rc;
    constexpr int smem_bytes = 1024 + (1 + 2 * KV_STAGES) * CH::tile_bytes(ATT_TILE) + 128;
    static_assert(smem_bytes <= 232448, "attention forward shared memory budget exceeded");
    auto kern = attn_fwd_kernel<HD, ALIBI>;
    static bool attr_set = false;
    if (!attr_set) {
        DOLO_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
        attr_set = true;
    }
    // upper bound on the number of q tiles without reading cu_seqlens on the host
    const int64_t max_tiles = (p.T + ATT_TILE - 1) / ATT_TILE + p.n_docs;
    DOLO_REQUIRE(max_tiles == p.n_tile_slots && max_tiles * p.n_heads < (1ll << 31), "attn_fwd: grid too large");
    dim3 grid((unsigned)(max_tiles * p.n_heads));
    kern<<<grid, FWD_THREADS, smem_bytes, st>>>(t64, tR, p);
    DOLO_LAUNCH_OK("attn_varlen_fwd");
    return DOLO_OK;
}

}  // namespace

uint32_t dolo_dropout_threshold(float p);  // dropout.cu

extern "C" int dolomite_b200_attn_varlen_fwd(const void* qkv, int64_t row_stride, void* out, float* lse,
                                             const int32_t* cu_seqlens, int n_docs, int64_t T, int max_seqlen,
                                             int n_groups, int q_per_group, int head_dim, float softmax_scale,
                                             void* stream) {
    return dolomite_b200_attn_varlen_fwd_dropout(qkv, row_stride, out, lse, cu_seqlens, n_docs, T, max_seqlen, n_groups,
                                                 q_per_group, head_dim, softmax_scale, 0.f, 0, 0, stream);
}

namespace {

// alibi_slopes == nullptr: the plain kernels
int attn_fwd(const void* qkv, int64_t row_stride, void* out, float* lse, const int32_t* cu_seqlens, int n_docs, int64_t T,
             int n_groups, int q_per_group, int head_dim, float softmax_scale, float dropout_p, uint32_t key0, uint32_t key1,
             const float* alibi_slopes, void* stream) {
    DOLO_REQUIRE(dropout_p >= 0.f && dropout_p < 1.f, "attn_fwd: dropout_p=%f must be in [0, 1)", double(dropout_p));
    DOLO_REQUIRE(n_docs >= 0 && T >= 0, "attn_fwd: negative sizes");
    if (T == 0 || n_docs == 0) return DOLO_OK;
    DOLO_REQUIRE(n_groups > 0 && q_per_group > 0, "attn_fwd: bad head grouping");
    DOLO_REQUIRE(row_stride % 8 == 0 && (reinterpret_cast<uintptr_t>(qkv) & 15) == 0, "attn_fwd: qkv alignment");
    DOLO_REQUIRE(int64_t(n_groups) * (q_per_group + 2) * head_dim <= row_stride, "attn_fwd: slot layout exceeds row");
    DOLO_REQUIRE(T < (1ll << 31), "attn_fwd: T too large");
    FwdParams p;
    p.out = static_cast<__nv_bfloat16*>(out);
    p.lse = lse;
    p.cu_seqlens = cu_seqlens;
    p.n_docs = n_docs;
    p.T = T;
    p.n_groups = n_groups;
    p.q_per_group = q_per_group;
    p.n_heads = n_groups * q_per_group;
    p.scale = softmax_scale;
    p.scale_log2 = softmax_scale * 1.4426950408889634f;
    p.drop.threshold = dolo_dropout_threshold(dropout_p);
    p.drop.keep_scale = 1.f / (1.f - dropout_p);
    p.drop.key0 = key0;
    p.drop.key1 = key1;
    p.n_tile_slots = int((T + ATT_TILE - 1) / ATT_TILE + n_docs);
    p.head_chunk = attn_head_chunk(dolo_option_attn_head_fastest(), p.n_heads, q_per_group);
    // all heads in one chunk when the K / V of the whole batch stay in L2 anyway (GQA / short batches): nothing to lose to
    // re-reads, and the longest-first order then spans every head
    if (p.head_chunk > 0 && T * int64_t(n_groups) * head_dim * 4 <= (24ll << 20)) p.head_chunk = p.n_heads;
    p.alibi_slopes = alibi_slopes;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const bool ab = alibi_slopes != nullptr;
    switch (head_dim) {
        case 16: return ab ? launch_fwd<16, true>(qkv, row_stride, p, st) : launch_fwd<16, false>(qkv, row_stride, p, st);
        case 32: return ab ? launch_fwd<32, true>(qkv, row_stride, p, st) : launch_fwd<32, false>(qkv, row_stride, p, st);
        case 64: return ab ? launch_fwd<64, true>(qkv, row_stride, p, st) : launch_fwd<64, false>(qkv, row_stride, p, st);
        case 80: return ab ? launch_fwd<80, true>(qkv, row_stride, p, st) : launch_fwd<80, false>(qkv, row_stride, p, st);
        case 96: return ab ? launch_fwd<96, true>(qkv, row_stride, p, st) : launch_fwd<96, false>(qkv, row_stride, p, st);
        case 128: return ab ? launch_fwd<128, true>(qkv, row_stride, p, st) : launch_fwd<128, false>(qkv, row_stride, p, st);
        case 160: case 192: case 256:
            return dolo_attn_wide_fwd(qkv, row_stride, out, lse, cu_seqlens, n_docs, T, n_groups, q_per_group, head_dim,
                                      softmax_scale, dropout_p, key0, key1, alibi_slopes, st);
        default: return dolo_set_error("attn_fwd: unsupported head_dim %d (supported: 16,32,64,80,96,128,160,192,256)", head_dim);
    }
}

}  // namespace

extern "C" int dolomite_b200_attn_varlen_fwd_dropout(const void* qkv, int64_t row_stride, void* out, float* lse,
                                                     const int32_t* cu_seqlens, int n_docs, int64_t T, int max_seqlen,
                                                     int n_groups, int q_per_group, int head_dim, float softmax_scale,
                                                     float dropout_p, uint32_t key0, uint32_t key1, void* stream) {
    (void)max_seqlen;
    return attn_fwd(qkv, row_stride, out, lse, cu_seqlens, n_docs, T, n_groups, q_per_group, head_dim, softmax_scale,
                    dropout_p, key0, key1, nullptr, stream);
}

extern "C" int dolomite_b200_attn_varlen_fwd_alibi(const void* qkv, int64_t row_stride, void* out, float* lse,
                                                   const int32_t* cu_seqlens, int n_docs, int64_t T, int max_seqlen,
                                                   int n_groups, int q_per_group, int head_dim, float softmax_scale,
                                                   float dropout_p, uint32_t key0, uint32_t key1,
                                                   const float* alibi_slopes, void* stream) {
    (void)max_seqlen;
    DOLO_REQUIRE(alibi_slopes != nullptr, "attn_fwd_alibi: alibi_slopes is null");
    return attn_fwd(qkv, row_stride, out, lse, cu_seqlens, n_docs, T, n_groups, q_per_group, head_dim, softmax_scale,
                    dropout_p, key0, key1, alibi_slopes, stream);
}
