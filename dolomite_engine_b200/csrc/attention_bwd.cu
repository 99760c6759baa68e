// Packed var-len causal attention backward on wgmma (autograd of flash_attn_varlen_func,
// attention/padding_free.py:51-62).
#include "attention_common.cuh"
#include "../../include/dolomite_b200.h"

using namespace dolo;

namespace {

struct BwdParams {
    const float* lse;      // [n_heads, T]
    const float* delta;    // [n_heads, T]
    __nv_bfloat16* dqkv;   // [T, row_stride]
    int64_t row_stride;
    const int32_t* cu_seqlens;
    int n_docs;
    int64_t T;
    int n_groups, q_per_group, n_heads;
    float scale, scale_log2;
    int head_chunk;    // CTA order (attention_common.cuh: attn_cta_order): kv groups per chunk, 0 = tiles fastest
    int head_chunk_q;  // the same for the query heads of the dQ kernel
    int n_tile_slots;  // upper bound of the number of 128-row key (dK/dV) or query (dQ) tiles of a head
    AttnDropout drop;  // attention-probability dropout of the forward being differentiated (threshold 0: none)
};

// Delta[h, t] = sum_d dO[t, h, d] * O[t, h, d].  Block = DELTA_TOK tokens: every thread takes 16-byte vectors of dO and O
// (coalesced over the whole [tokens, heads*hd] slab) and leaves its 8-product partial in shared memory; the partials of a
// head are then summed in a fixed order (deterministic) and written token-fastest, so each head's DELTA_TOK floats fill
// one 32-byte sector.
constexpr int DELTA_TOK = 8;
__global__ void __launch_bounds__(256)
    attn_delta_kernel(const uint4* __restrict__ dout, const uint4* __restrict__ out, float* __restrict__ delta, int64_t T,
                      int n_heads, int vec_per_head) {
    extern __shared__ float part[];  // [DELTA_TOK][n_heads * vec_per_head]
    const int64_t t0 = int64_t(blockIdx.x) * DELTA_TOK;
    const int ntok = (T - t0) < DELTA_TOK ? int(T - t0) : DELTA_TOK;
    const int vec_per_tok = n_heads * vec_per_head;
    const int total = ntok * vec_per_tok;
    const uint4* a = dout + t0 * vec_per_tok;
    const uint4* b = out + t0 * vec_per_tok;
    for (int i = threadIdx.x; i < total; i += blockDim.x) {
        const uint4 x = __ldg(a + i), y = __ldg(b + i);
        float s = bf16_lo(x.x) * bf16_lo(y.x) + bf16_hi(x.x) * bf16_hi(y.x);
        s += bf16_lo(x.y) * bf16_lo(y.y) + bf16_hi(x.y) * bf16_hi(y.y);
        s += bf16_lo(x.z) * bf16_lo(y.z) + bf16_hi(x.z) * bf16_hi(y.z);
        s += bf16_lo(x.w) * bf16_lo(y.w) + bf16_hi(x.w) * bf16_hi(y.w);
        part[i] = s;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n_heads * DELTA_TOK; i += blockDim.x) {
        const int h = i / DELTA_TOK, tl = i - h * DELTA_TOK;
        if (tl < ntok) {
            const float* p = part + tl * vec_per_tok + h * vec_per_head;
            float s = 0.f;
            for (int k = 0; k < vec_per_head; ++k) s += p[k];
            delta[int64_t(h) * T + t0 + tl] = s;
        }
    }
}

// One CTA = one 128-row key/value tile of one kv-head group of one document, two warpgroups of 64 key rows each; it loops
// over the query heads of the group and the 64-row query tiles that see the key tile (causal) and keeps dK_j, dV_j
// accumulating in registers.  Everything is computed in the "transposed" frame (accumulator row == key row) so that P^T and
// dS^T feed the tensor core straight from registers as the A operand.  Per step, every warpgroup runs
//     S^T  = K_j Q_i^T            (SS)           dP^T = V_j dO_i^T             (SS)
//     P^T  = exp2(S^T*scale - LSE_i) ,  dS^T = scale * P^T o (dP^T - Delta_i)     (registers)
//     dV_j += P^T dO_i            (RS, B = dO MN-major)
//     dK_j += dS^T Q_i            (RS, B = Q  MN-major)
// Thread 0 also issues the TMA loads (K_j, V_j once; Q_i, dO_i through a 2-stage ring).
// dQ has its own kernel (attn_dq_kernel below: one CTA per query tile walks the key tiles in order), so that every
// gradient is summed in a fixed order and the backward is bit-identical from run to run -- adding the dQ contributions
// of the key-tile CTAs with atomics would not be.
constexpr int BWD_THREADS = 256;
constexpr int BWD_QT = 64;  // query rows per step
constexpr int QDO_STAGES = 2;

template <int HD>
__global__ void __launch_bounds__(BWD_THREADS, 1)
    attn_bwd_kernel(const __grid_constant__ CUtensorMap tq64, const __grid_constant__ CUtensorMap tqR,
                    const __grid_constant__ CUtensorMap to64, const __grid_constant__ CUtensorMap toR, const BwdParams p) {
    using CH = HeadChunks<HD>;
    constexpr int KV_BYTES = CH::tile_bytes(ATT_TILE);
    constexpr int QT_BYTES = CH::tile_bytes(BWD_QT);

    int cta_tile, group;  // key tiles of a document in natural order = longest first
    attn_cta_order(p.head_chunk, p.n_tile_slots, cta_tile, group);
    const TileLoc loc = locate_tile(p.cu_seqlens, p.n_docs, cta_tile);
    if (!loc.valid) return;
    const int k0 = loc.tile * ATT_TILE;             // first key (doc-relative) of this tile
    const int i0 = k0 / BWD_QT;                     // first query tile that sees a key of the tile
    const int n_qt = (loc.doc_len + BWD_QT - 1) / BWD_QT;
    const int n_i = n_qt - i0;
    const int n_steps = n_i * p.q_per_group;
    const int k_col = (group * (p.q_per_group + 2) + p.q_per_group) * HD;
    const int v_col = k_col + HD;

    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_align_1024(smem_raw);
    uint8_t* sK = smem;
    uint8_t* sV = sK + KV_BYTES;
    uint8_t* sQ = sV + KV_BYTES;                // [QDO_STAGES]
    uint8_t* sO = sQ + QDO_STAGES * QT_BYTES;   // [QDO_STAGES] dO
    uint64_t* bars = reinterpret_cast<uint64_t*>(sO + QDO_STAGES * QT_BYTES);
    uint64_t* kv_full = bars;       // 1
    uint64_t* qd_full = bars + 1;   // [QDO_STAGES]
    uint64_t* qd_empty = bars + 3;  // [QDO_STAGES], one arrive per warp

    const int wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    auto load_step = [&](int n, int s) {
        const int hl = n / n_i, qi = i0 + n % n_i;
        const int head = group * p.q_per_group + hl;
        const int q_col = (group * (p.q_per_group + 2) + hl) * HD;
        mbar_expect_tx(&qd_full[s], 2 * QT_BYTES);
        tma_load_chunked<HD, BWD_QT>(sQ + s * QT_BYTES, &tq64, &tqR, &qd_full[s], q_col, loc.doc_start + qi * BWD_QT);
        tma_load_chunked<HD, BWD_QT>(sO + s * QT_BYTES, &to64, &toR, &qd_full[s], head * HD, loc.doc_start + qi * BWD_QT);
    };
    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tq64);
        tma_prefetch_desc(&to64);
        if (CH::REM > 0) {
            tma_prefetch_desc(&tqR);
            tma_prefetch_desc(&toR);
        }
        mbar_init(kv_full, 1);
        for (int i = 0; i < QDO_STAGES; ++i) {
            mbar_init(&qd_full[i], 1);
            mbar_init(&qd_empty[i], BWD_THREADS / 32);
        }
        mbar_fence_init();
        mbar_expect_tx(kv_full, 2 * KV_BYTES);
        tma_load_chunked<HD, ATT_TILE>(sK, &tq64, &tqR, kv_full, k_col, loc.doc_start + k0);
        tma_load_chunked<HD, ATT_TILE>(sV, &tq64, &tqR, kv_full, v_col, loc.doc_start + k0);
        for (int n = 0; n < QDO_STAGES && n < n_steps; ++n) load_step(n, n);
    }
    __syncthreads();

    const int wr = (warp & 3) * 16 + (lane >> 2);  // first of the two accumulator rows of this thread (and wr + 8)
    const int wc = 2 * (lane & 3);                 // first accumulator column inside each n8 block
    const int kr[2] = {k0 + wg * 64 + wr, k0 + wg * 64 + wr + 8};  // doc-relative keys of the two rows
    const bool drop = p.drop.threshold != 0;
    const float log2e = 1.4426950408889634f;
    const uint32_t sk = smem_u32(sK) , sv = smem_u32(sV);

    float dv[HD / 2], dk[HD / 2];
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) dv[i] = dk[i] = 0.f;

    mbar_wait(kv_full, 0, 30);
    for (int n = 0; n < n_steps; ++n) {
        const int s = n & (QDO_STAGES - 1);
        const int hl = n / n_i, qi = i0 + n % n_i;
        const int head = group * p.q_per_group + hl;
        const int q0 = qi * BWD_QT;
        const uint32_t head_key = dropout_head_key(uint32_t(head), p.drop.key0, p.drop.key1);
        // LSE / Delta of this thread's 16 query columns
        float lse_c[BWD_QT / 8][2], del_c[BWD_QT / 8][2];
#pragma unroll
        for (int b = 0; b < BWD_QT / 8; ++b)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int q = q0 + 8 * b + wc + e;
                const int64_t idx = int64_t(head) * p.T + loc.doc_start + q;
                lse_c[b][e] = q < loc.doc_len ? __ldg(p.lse + idx) * log2e : 0.f;
                del_c[b][e] = q < loc.doc_len ? __ldg(p.delta + idx) : 0.f;
            }
        mbar_wait(&qd_full[s], (n / QDO_STAGES) & 1, 31);
        const uint32_t sq = smem_u32(sQ + s * QT_BYTES), so = smem_u32(sO + s * QT_BYTES);

        float st[BWD_QT / 2], dpt[BWD_QT / 2];
        wgmma_fence();
#pragma unroll
        for (int c = 0; c < CH::NCHUNK; ++c) {
            const int w = CH::width(c);
            const uint32_t krow = CH::offset(c, ATT_TILE) + wg * 64 * 2 * w;  // this warpgroup's 64 key rows of the chunk
#pragma unroll
            for (int k = 0; k < w / 16; ++k) {
                wgmma_ss<BWD_QT, 0, 0>(st, chunk_desc_kmajor(sk + krow, w, k), chunk_desc_kmajor(sq + CH::offset(c, BWD_QT), w, k),
                                       (c != 0 || k != 0) ? 1u : 0u);
                wgmma_ss<BWD_QT, 0, 0>(dpt, chunk_desc_kmajor(sv + krow, w, k), chunk_desc_kmajor(so + CH::offset(c, BWD_QT), w, k),
                                       (c != 0 || k != 0) ? 1u : 0u);
            }
        }
        wgmma_commit();
        wgmma_wait<0>();
        reg_fence<BWD_QT / 2>(st);
        reg_fence<BWD_QT / 2>(dpt);

        // ---------------- P^T, dS^T ----------------
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int b = 0; b < BWD_QT / 8; ++b)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int q = q0 + 8 * b + wc + e;
                    const int i = 4 * b + 2 * h + e;
                    const bool ok = q >= kr[h] && q < loc.doc_len;  // causal, and a real query of the document
                    float pr = ok ? fast_exp2(fmaf(st[i], p.scale_log2, -lse_c[b][e])) : 0.f;
                    float dp = dpt[i];
                    if (drop) {
                        const float z = attn_drop_scale(p.drop, head_key, loc.doc_start + q, loc.doc_start + kr[h]);
                        dp *= z;
                        st[i] = pr * z;  // dropped-and-rescaled probabilities: what dV sees
                    } else {
                        st[i] = pr;
                    }
                    dpt[i] = p.scale * pr * (dp - del_c[b][e]);
                }
        uint32_t pa[BWD_QT / 16][4], da[BWD_QT / 16][4];
#pragma unroll
        for (int kk = 0; kk < BWD_QT / 16; ++kk) {
            acc_to_a_frag(st, kk, pa[kk]);
            acc_to_a_frag(dpt, kk, da[kk]);
        }

        // ---------------- dV += P^T dO,  dK += dS^T Q ----------------
        wgmma_fence();
#pragma unroll
        for (int c = 0; c < CH::NCHUNK; ++c) {
#pragma unroll
            for (int kk = 0; kk < BWD_QT / 16; ++kk) {
                if (CH::width(c) == 64) {
                    wgmma_rs<64, 1>(dv + CH::col(c) / 2, pa[kk], chunk_desc_mnmajor(so + CH::offset(c, BWD_QT), 64, kk), 1u);
                    wgmma_rs<64, 1>(dk + CH::col(c) / 2, da[kk], chunk_desc_mnmajor(sq + CH::offset(c, BWD_QT), 64, kk), 1u);
                } else {
                    constexpr int R = CH::REM ? CH::REM : 16;
                    wgmma_rs<R, 1>(dv + CH::col(c) / 2, pa[kk], chunk_desc_mnmajor(so + CH::offset(c, BWD_QT), R, kk), 1u);
                    wgmma_rs<R, 1>(dk + CH::col(c) / 2, da[kk], chunk_desc_mnmajor(sq + CH::offset(c, BWD_QT), R, kk), 1u);
                }
            }
        }
        wgmma_commit();

        wgmma_wait<0>();
        reg_fence<HD / 2>(dv);
        reg_fence<HD / 2>(dk);
        if (lane == 0) mbar_arrive(&qd_empty[s]);  // Q_i / dO_i of this warp's MMAs are read
        if (threadIdx.x == 0 && n + QDO_STAGES < n_steps) {
            mbar_wait(&qd_empty[s], (n / QDO_STAGES) & 1, 32);
            load_step(n + QDO_STAGES, s);
        }
        __syncwarp();
    }

    // ---------------- dK_j, dV_j -> the k / v slots of dqkv ----------------
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        if (kr[h] >= loc.doc_len) continue;
        __nv_bfloat16* row = p.dqkv + (loc.doc_start + int64_t(kr[h])) * p.row_stride;
#pragma unroll
        for (int b = 0; b < HD / 8; ++b) {
            *reinterpret_cast<uint32_t*>(row + k_col + 8 * b + wc) = pack_bf16(dk[4 * b + 2 * h], dk[4 * b + 2 * h + 1]);
            *reinterpret_cast<uint32_t*>(row + v_col + 8 * b + wc) = pack_bf16(dv[4 * b + 2 * h], dv[4 * b + 2 * h + 1]);
        }
    }
}

template <int HD>
int launch_bwd(const void* dout, const void* qkv, int64_t row_stride, const BwdParams& p, cudaStream_t st) {
    using CH = HeadChunks<HD>;
    CUtensorMap tq64, tqR, to64, toR;
    int rc = attn_make_maps<HD>(qkv, row_stride, p.T, &tq64, &tqR);
    if (rc) return rc;
    rc = attn_make_maps<HD>(dout, int64_t(p.n_heads) * HD, p.T, &to64, &toR);
    if (rc) return rc;
    constexpr int smem_bytes = 1024 + 2 * CH::tile_bytes(ATT_TILE) + 2 * QDO_STAGES * CH::tile_bytes(BWD_QT) + 128;
    static_assert(smem_bytes <= 232448, "attention backward shared memory budget exceeded");
    auto kern = attn_bwd_kernel<HD>;
    static bool attr_set = false;
    if (!attr_set) {
        DOLO_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
        attr_set = true;
    }
    const int64_t max_tiles = (p.T + ATT_TILE - 1) / ATT_TILE + p.n_docs;
    DOLO_REQUIRE(max_tiles == p.n_tile_slots && max_tiles * p.n_groups < (1ll << 31), "attn_bwd: grid too large");
    dim3 grid((unsigned)(max_tiles * p.n_groups));
    kern<<<grid, BWD_THREADS, smem_bytes, st>>>(tq64, tqR, to64, toR, p);
    DOLO_LAUNCH_OK("attn_varlen_bwd");
    return DOLO_OK;
}

// dQ of the backward: one CTA = one 128-row query tile of one head of one document, two warpgroups of 64 queries each,
// looping over the 64-row key tiles the queries see, in order.  Per key tile every warpgroup recomputes
//     S  = Q_i K_j^T ,  dP = dO_i V_j^T           (SS)
//     dS = scale * P o (dP - Delta_i)             (registers, P = exp2(S*scale - LSE_i))
//     dQ_i += dS K_j                              (RS, B = K MN-major)
// and finally writes dQ_i (bf16) into the q slots of dqkv.  Thread 0 issues the TMA loads: Q_i and dO_i once, (K_j, V_j)
// through a 2-stage ring.
constexpr int DQ_THREADS = 256;
constexpr int DQ_KT = 64;  // keys per step

template <int HD>
__global__ void __launch_bounds__(DQ_THREADS, 1)
    attn_dq_kernel(const __grid_constant__ CUtensorMap tq64, const __grid_constant__ CUtensorMap tqR,
                   const __grid_constant__ CUtensorMap to64, const __grid_constant__ CUtensorMap toR, const BwdParams p) {
    using CH = HeadChunks<HD>;
    constexpr int Q_BYTES = CH::tile_bytes(ATT_TILE);
    constexpr int KT_BYTES = CH::tile_bytes(DQ_KT);

    int ti, head;
    attn_cta_order(p.head_chunk_q, p.n_tile_slots, ti, head);
    ti = p.n_tile_slots - 1 - ti;  // long (late) tiles first
    const TileLoc loc = locate_tile(p.cu_seqlens, p.n_docs, ti);
    if (!loc.valid) return;
    const int group = head / p.q_per_group, slot = head % p.q_per_group;
    const int q_col = (group * (p.q_per_group + 2) + slot) * HD;
    const int k_col = (group * (p.q_per_group + 2) + p.q_per_group) * HD;
    const int v_col = k_col + HD;
    const int q0 = loc.tile * ATT_TILE;
    const int k_end = min(q0 + ATT_TILE, loc.doc_len);  // causal: keys [0, k_end) are seen by some query of the tile
    const int n_kt = (k_end + DQ_KT - 1) / DQ_KT;

    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_align_1024(smem_raw);
    uint8_t* sQ = smem;
    uint8_t* sO = sQ + Q_BYTES;       // dO
    uint8_t* sK = sO + Q_BYTES;       // [2]
    uint8_t* sV = sK + 2 * KT_BYTES;  // [2]
    uint64_t* bars = reinterpret_cast<uint64_t*>(sV + 2 * KT_BYTES);
    uint64_t* q_full = bars;        // 1
    uint64_t* kv_full = bars + 1;   // [2]
    uint64_t* kv_empty = bars + 3;  // [2], one arrive per warp

    const int wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    auto load_kv = [&](int j, int s) {
        mbar_expect_tx(&kv_full[s], 2 * KT_BYTES);
        tma_load_chunked<HD, DQ_KT>(sK + s * KT_BYTES, &tq64, &tqR, &kv_full[s], k_col, loc.doc_start + j * DQ_KT);
        tma_load_chunked<HD, DQ_KT>(sV + s * KT_BYTES, &tq64, &tqR, &kv_full[s], v_col, loc.doc_start + j * DQ_KT);
    };
    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tq64);
        tma_prefetch_desc(&to64);
        if (CH::REM > 0) {
            tma_prefetch_desc(&tqR);
            tma_prefetch_desc(&toR);
        }
        mbar_init(q_full, 1);
        for (int i = 0; i < 2; ++i) {
            mbar_init(&kv_full[i], 1);
            mbar_init(&kv_empty[i], DQ_THREADS / 32);
        }
        mbar_fence_init();
        mbar_expect_tx(q_full, 2 * Q_BYTES);
        tma_load_chunked<HD, ATT_TILE>(sQ, &tq64, &tqR, q_full, q_col, loc.doc_start + q0);
        tma_load_chunked<HD, ATT_TILE>(sO, &to64, &toR, q_full, head * HD, loc.doc_start + q0);
        for (int j = 0; j < 2 && j < n_kt; ++j) load_kv(j, j);
    }
    __syncthreads();

    const int wr = (warp & 3) * 16 + (lane >> 2);
    const int wc = 2 * (lane & 3);
    const int qr[2] = {q0 + wg * 64 + wr, q0 + wg * 64 + wr + 8};  // doc-relative queries of the two rows
    const bool drop = p.drop.threshold != 0;
    const uint32_t head_key = dropout_head_key(uint32_t(head), p.drop.key0, p.drop.key1);
    const float log2e = 1.4426950408889634f;
    float lse_r[2], del_r[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const bool ok = qr[h] < loc.doc_len;
        const int64_t idx = int64_t(head) * p.T + loc.doc_start + qr[h];
        lse_r[h] = ok ? __ldg(p.lse + idx) * log2e : 0.f;
        del_r[h] = ok ? __ldg(p.delta + idx) : 0.f;
    }
    const uint32_t sq = smem_u32(sQ), so = smem_u32(sO);
    float dq[HD / 2];
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) dq[i] = 0.f;

    mbar_wait(q_full, 0, 40);
    for (int j = 0; j < n_kt; ++j) {
        const int s = j & 1;
        mbar_wait(&kv_full[s], (j >> 1) & 1, 41);
        const uint32_t sk = smem_u32(sK + s * KT_BYTES), sv = smem_u32(sV + s * KT_BYTES);
        float sc[DQ_KT / 2], dp[DQ_KT / 2];
        wgmma_fence();
#pragma unroll
        for (int c = 0; c < CH::NCHUNK; ++c) {
            const int w = CH::width(c);
            const uint32_t qrow = CH::offset(c, ATT_TILE) + wg * 64 * 2 * w;  // this warpgroup's 64 query rows of the chunk
#pragma unroll
            for (int k = 0; k < w / 16; ++k) {
                wgmma_ss<DQ_KT, 0, 0>(sc, chunk_desc_kmajor(sq + qrow, w, k), chunk_desc_kmajor(sk + CH::offset(c, DQ_KT), w, k),
                                      (c != 0 || k != 0) ? 1u : 0u);
                wgmma_ss<DQ_KT, 0, 0>(dp, chunk_desc_kmajor(so + qrow, w, k), chunk_desc_kmajor(sv + CH::offset(c, DQ_KT), w, k),
                                      (c != 0 || k != 0) ? 1u : 0u);
            }
        }
        wgmma_commit();
        wgmma_wait<0>();
        reg_fence<DQ_KT / 2>(sc);
        reg_fence<DQ_KT / 2>(dp);

#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int b = 0; b < DQ_KT / 8; ++b)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int k = j * DQ_KT + 8 * b + wc + e;
                    const int i = 4 * b + 2 * h + e;
                    const bool ok = k <= qr[h] && qr[h] < loc.doc_len;  // causal, and a real query of the document
                    const float pr = ok ? fast_exp2(fmaf(sc[i], p.scale_log2, -lse_r[h])) : 0.f;
                    float d = dp[i];
                    if (drop) d *= attn_drop_scale(p.drop, head_key, loc.doc_start + qr[h], loc.doc_start + k);
                    sc[i] = p.scale * pr * (d - del_r[h]);
                }
        uint32_t da[DQ_KT / 16][4];
#pragma unroll
        for (int kk = 0; kk < DQ_KT / 16; ++kk) acc_to_a_frag(sc, kk, da[kk]);

        wgmma_fence();
#pragma unroll
        for (int c = 0; c < CH::NCHUNK; ++c) {
#pragma unroll
            for (int kk = 0; kk < DQ_KT / 16; ++kk) {
                if (CH::width(c) == 64) {
                    wgmma_rs<64, 1>(dq + CH::col(c) / 2, da[kk], chunk_desc_mnmajor(sk + CH::offset(c, DQ_KT), 64, kk), 1u);
                } else {
                    constexpr int R = CH::REM ? CH::REM : 16;
                    wgmma_rs<R, 1>(dq + CH::col(c) / 2, da[kk], chunk_desc_mnmajor(sk + CH::offset(c, DQ_KT), R, kk), 1u);
                }
            }
        }
        wgmma_commit();
        wgmma_wait<0>();
        reg_fence<HD / 2>(dq);
        if (lane == 0) mbar_arrive(&kv_empty[s]);
        if (threadIdx.x == 0 && j + 2 < n_kt) {
            mbar_wait(&kv_empty[s], (j >> 1) & 1, 42);  // both warpgroups are done with key tile j
            load_kv(j + 2, s);
        }
        __syncwarp();
    }

#pragma unroll
    for (int h = 0; h < 2; ++h) {
        if (qr[h] >= loc.doc_len) continue;
        __nv_bfloat16* row = p.dqkv + (loc.doc_start + int64_t(qr[h])) * p.row_stride + q_col + wc;
#pragma unroll
        for (int b = 0; b < HD / 8; ++b)
            *reinterpret_cast<uint32_t*>(row + 8 * b) = pack_bf16(dq[4 * b + 2 * h], dq[4 * b + 2 * h + 1]);
    }
}

template <int HD>
int launch_dq(const void* dout, const void* qkv, int64_t row_stride, const BwdParams& p, cudaStream_t st) {
    using CH = HeadChunks<HD>;
    CUtensorMap tq64, tqR, to64, toR;
    int rc = attn_make_maps<HD>(qkv, row_stride, p.T, &tq64, &tqR);
    if (rc) return rc;
    rc = attn_make_maps<HD>(dout, int64_t(p.n_heads) * HD, p.T, &to64, &toR);
    if (rc) return rc;
    constexpr int smem_bytes = 1024 + 2 * CH::tile_bytes(ATT_TILE) + 4 * CH::tile_bytes(DQ_KT) + 128;
    static_assert(smem_bytes <= 232448, "attention dQ shared memory budget exceeded");
    auto kern = attn_dq_kernel<HD>;
    static bool attr_set = false;
    if (!attr_set) {
        DOLO_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
        attr_set = true;
    }
    const int64_t max_tiles = (p.T + ATT_TILE - 1) / ATT_TILE + p.n_docs;
    DOLO_REQUIRE(max_tiles == p.n_tile_slots && max_tiles * p.n_heads < (1ll << 31), "attn_bwd: grid too large");
    dim3 grid((unsigned)(max_tiles * p.n_heads));
    kern<<<grid, DQ_THREADS, smem_bytes, st>>>(tq64, tqR, to64, toR, p);
    DOLO_LAUNCH_OK("attn_varlen_bwd_dq");
    return DOLO_OK;
}

inline int64_t align256(int64_t x) { return (x + 255) & ~int64_t(255); }

}  // namespace

extern "C" int64_t dolomite_b200_attn_varlen_bwd_workspace_bytes(int64_t T, int n_groups, int q_per_group,
                                                                 int head_dim) {
    const int64_t nh = int64_t(n_groups) * q_per_group;
    (void)head_dim;
    return align256(nh * T * 4) + 256;  // Delta
}

uint32_t dolo_dropout_threshold(float p);  // dropout.cu

extern "C" int dolomite_b200_attn_varlen_bwd(const void* dout, const void* qkv, int64_t row_stride, const void* out,
                                             const float* lse, void* dqkv, const int32_t* cu_seqlens, int n_docs,
                                             int64_t T, int max_seqlen, int n_groups, int q_per_group, int head_dim,
                                             float softmax_scale, void* workspace, void* stream) {
    return dolomite_b200_attn_varlen_bwd_dropout(dout, qkv, row_stride, out, lse, dqkv, cu_seqlens, n_docs, T, max_seqlen,
                                                 n_groups, q_per_group, head_dim, softmax_scale, 0.f, 0, 0, workspace, stream);
}

extern "C" int dolomite_b200_attn_varlen_bwd_dropout(const void* dout, const void* qkv, int64_t row_stride, const void* out,
                                                     const float* lse, void* dqkv, const int32_t* cu_seqlens, int n_docs,
                                                     int64_t T, int max_seqlen, int n_groups, int q_per_group,
                                                     int head_dim, float softmax_scale, float dropout_p, uint32_t key0,
                                                     uint32_t key1, void* workspace, void* stream) {
    (void)max_seqlen;
    DOLO_REQUIRE(dropout_p >= 0.f && dropout_p < 1.f, "attn_bwd: dropout_p=%f must be in [0, 1)", double(dropout_p));
    if (T == 0 || n_docs == 0) return DOLO_OK;
    DOLO_REQUIRE(n_groups > 0 && q_per_group > 0, "attn_bwd: bad head grouping");
    DOLO_REQUIRE(row_stride % 8 == 0 && (reinterpret_cast<uintptr_t>(qkv) & 15) == 0 &&
                     (reinterpret_cast<uintptr_t>(dqkv) & 15) == 0 && (reinterpret_cast<uintptr_t>(dout) & 15) == 0,
                 "attn_bwd: alignment");
    DOLO_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "attn_bwd: workspace must be 256-byte aligned");
    DOLO_REQUIRE(T < (1ll << 31), "attn_bwd: T too large");
    const int nh = n_groups * q_per_group;
    DOLO_REQUIRE(int64_t(nh) * T < (1ll << 31), "attn_bwd: heads * T too large for the dQ tile reduce");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    float* delta = static_cast<float*>(workspace);
    {
        const int64_t blocks = (T + DELTA_TOK - 1) / DELTA_TOK;
        attn_delta_kernel<<<(unsigned)blocks, 256, size_t(nh) * (head_dim / 8) * DELTA_TOK * sizeof(float), st>>>(
            static_cast<const uint4*>(dout), static_cast<const uint4*>(out), delta, T, nh, head_dim / 8);
        DOLO_LAUNCH_OK("attn_delta");
    }
    BwdParams p;
    p.lse = lse;
    p.delta = delta;
    p.dqkv = static_cast<__nv_bfloat16*>(dqkv);
    p.row_stride = row_stride;
    p.cu_seqlens = cu_seqlens;
    p.n_docs = n_docs;
    p.T = T;
    p.n_groups = n_groups;
    p.q_per_group = q_per_group;
    p.n_heads = nh;
    p.scale = softmax_scale;
    p.scale_log2 = softmax_scale * 1.4426950408889634f;
    p.n_tile_slots = int((T + ATT_TILE - 1) / ATT_TILE + n_docs);
    p.head_chunk = attn_head_chunk(dolo_option_attn_head_fastest(), n_groups, 1);
    p.head_chunk_q = attn_head_chunk(dolo_option_attn_head_fastest(), nh, q_per_group);
    p.drop.threshold = dolo_dropout_threshold(dropout_p);
    p.drop.keep_scale = 1.f / (1.f - dropout_p);
    p.drop.key0 = key0;
    p.drop.key1 = key1;
    int rc;
    switch (head_dim) {
        case 16: rc = launch_bwd<16>(dout, qkv, row_stride, p, st); if (!rc) rc = launch_dq<16>(dout, qkv, row_stride, p, st); break;
        case 32: rc = launch_bwd<32>(dout, qkv, row_stride, p, st); if (!rc) rc = launch_dq<32>(dout, qkv, row_stride, p, st); break;
        case 64: rc = launch_bwd<64>(dout, qkv, row_stride, p, st); if (!rc) rc = launch_dq<64>(dout, qkv, row_stride, p, st); break;
        case 80: rc = launch_bwd<80>(dout, qkv, row_stride, p, st); if (!rc) rc = launch_dq<80>(dout, qkv, row_stride, p, st); break;
        case 96: rc = launch_bwd<96>(dout, qkv, row_stride, p, st); if (!rc) rc = launch_dq<96>(dout, qkv, row_stride, p, st); break;
        case 128: rc = launch_bwd<128>(dout, qkv, row_stride, p, st); if (!rc) rc = launch_dq<128>(dout, qkv, row_stride, p, st); break;
        default: return dolo_set_error("attn_bwd: unsupported head_dim %d (supported: 16,32,64,80,96,128)", head_dim);
    }
    if (rc) return rc;
    return DOLO_OK;
}
