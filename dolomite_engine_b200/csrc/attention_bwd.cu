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
    const float* alibi_slopes;  // [n_heads] fp32, read by the ALIBI instances only
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

// Both kernels below are warp-specialised (384 threads): warpgroup 0 is the producer and keeps only ATT_PRODUCER_REGS
// registers per thread; warpgroups 1 and 2 are the consumers, each owning 64 rows of the CTA's 128-row tile.  One elected
// producer thread is the only one that waits on `empty` barriers and issues the TMA loads of the ring, so no consumer ever
// waits for the other: the two consumer warpgroups drift apart and one's elementwise phase overlaps the other's MMAs.
constexpr int ATT_BWD_THREADS = 384;
constexpr int ATT_PRODUCER_REGS = 24;
constexpr int ATT_CONSUMER_REGS = 240;
static_assert(ATT_PRODUCER_REGS * 128 + 2 * ATT_CONSUMER_REGS * 128 <= 65536, "register file exceeded");

// One CTA = one 128-row key/value tile of one kv-head group of one document; it loops over the query heads of the group and
// the 64-row query tiles that see the key tile (causal) and keeps dK_j, dV_j accumulating in registers.  Everything is
// computed in the "transposed" frame (accumulator row == key row) so that P^T and dS^T feed the tensor core straight from
// registers as the A operand.  Per step, every consumer warpgroup (64 key rows) runs
//     S^T  = K_j Q_i^T            (SS)           dP^T = V_j dO_i^T             (SS)
//     P^T  = exp2(S^T*scale - LSE_i) ,  dS^T = scale * P^T o (dP^T - Delta_i)     (registers)
//     dV_j += P^T dO_i            (RS, B = dO MN-major)
//     dK_j += dS^T Q_i            (RS, B = Q  MN-major)
// Producer: thread 0 loads K_j, V_j once; an elected lane of warp 0 streams Q_i, dO_i through a QDO_STAGES-deep ring and
// warp 1 stages the 64 LSE_i (times log2 e) and Delta_i values of each step into the same ring stage with plain loads (the
// rows of a document start anywhere, so they are not bulk-copy aligned); both arrive on the stage's `full` barrier.
// Only the steps whose query tile reaches a key row of the warpgroup (qi <= i0 + cw) or crosses the document end test the
// causal / bounds predicate; the interior steps run the bare formula.  The MMAs of a step run in the serial order SS ->
// elementwise -> RS: issuing the next step's SS group behind the RS group makes ptxas serialise every wgmma of the kernel.
// ALIBI: P^T = exp2(log2(e) * (S^T*scale + bias_k) - LSE_i), the bias of the forward (one per key row of the thread); the
// bias has no gradient, so dS^T is unchanged.
// dQ has its own kernel (attn_dq_kernel below: one CTA per query tile walks the key tiles in order), so that every
// gradient is summed in a fixed order and the backward is bit-identical from run to run -- adding the dQ contributions
// of the key-tile CTAs with atomics would not be.
constexpr int BWD_QT = 64;  // query rows per step
// opaque, mbar_spin and mbar_arrive_lane0: attention_common.cuh
constexpr int QDO_STAGES = 4;

// P^T (into st) and dS^T (into dpt) of one step from S^T, dP^T; MASK = test causality and the document end per element
template <bool ALIBI, bool MASK>
__device__ __forceinline__ void bwd_p_ds(float (&st)[BWD_QT / 2], float (&dpt)[BWD_QT / 2], const float* ls, const float* ds,
                                         const BwdParams& p, const TileLoc& loc, int q0, int wc, const int (&kr)[2], int head,
                                         uint32_t head_key, bool drop) {
    // ALIBI: log2(e) * bias of the key row
    const float slope = ALIBI ? __ldg(p.alibi_slopes + head) : 0.f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const float bias_r = ALIBI ? attn_alibi_bias(slope, kr[h]) * ATT_LOG2E : 0.f;
#pragma unroll
        for (int b = 0; b < BWD_QT / 8; ++b) {
            const float2 l = *reinterpret_cast<const float2*>(ls + 8 * b + wc);
            const float2 d = *reinterpret_cast<const float2*>(ds + 8 * b + wc);
            const float lse_c[2] = {l.x, l.y}, del_c[2] = {d.x, d.y};
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int q = q0 + 8 * b + wc + e;
                const int i = 4 * b + 2 * h + e;
                const bool ok = !MASK || (q >= kr[h] && q < loc.doc_len);  // causal, and a real query of the document
                float pr;
                if constexpr (ALIBI)
                    pr = ok ? fast_exp2(fmaf(st[i], p.scale_log2, bias_r) - lse_c[e]) : 0.f;
                else
                    pr = ok ? fast_exp2(fmaf(st[i], p.scale_log2, -lse_c[e])) : 0.f;
                float dp = dpt[i];
                if (drop) {
                    const float z = attn_drop_scale(p.drop, head_key, loc.doc_start + q, loc.doc_start + kr[h]);
                    dp *= z;
                    st[i] = pr * z;  // dropped-and-rescaled probabilities: what dV sees
                } else {
                    st[i] = pr;
                }
                dpt[i] = p.scale * pr * (dp - del_c[e]);
            }
        }
    }
}

template <int HD, bool ALIBI>
__global__ void __launch_bounds__(ATT_BWD_THREADS, 1)
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
    float* sL = reinterpret_cast<float*>(sO + QDO_STAGES * QT_BYTES);  // [QDO_STAGES][LSE * log2 e, Delta][BWD_QT]
    uint64_t* bars = reinterpret_cast<uint64_t*>(sL + QDO_STAGES * 2 * BWD_QT);
    uint64_t* kv_full = bars;                    // 1
    uint64_t* qd_full = bars + 1;                // [QDO_STAGES]: TMA bytes + one arrive per lane of producer warp 1
    uint64_t* qd_empty = bars + 1 + QDO_STAGES;  // [QDO_STAGES], one arrive per consumer warp

    const int wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const float log2e = 1.4426950408889634f;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tq64);
        tma_prefetch_desc(&to64);
        if (CH::REM > 0) {
            tma_prefetch_desc(&tqR);
            tma_prefetch_desc(&toR);
        }
        mbar_init(kv_full, 1);
        for (int i = 0; i < QDO_STAGES; ++i) {
            mbar_init(&qd_full[i], 1 + 32);
            mbar_init(&qd_empty[i], 8);
        }
        mbar_fence_init();
        mbar_expect_tx(kv_full, 2 * KV_BYTES);
        tma_load_chunked<HD, ATT_TILE>(sK, &tq64, &tqR, kv_full, k_col, loc.doc_start + k0);
        tma_load_chunked<HD, ATT_TILE>(sV, &tq64, &tqR, kv_full, v_col, loc.doc_start + k0);
    }
    __syncthreads();

    if (wg == 0) {
        // ================= producer =================
        setmaxnreg_dec<ATT_PRODUCER_REGS>();  // all four warps, before warps 2, 3 leave
        if (warp == 0) {
            if (elect_one()) {
                int s = 0;
                uint32_t ph = 0;
                for (int n = 0; n < n_steps; ++n) {
                    const int hl = n / n_i, qi = i0 + n % n_i;
                    const int q_col = (group * (p.q_per_group + 2) + hl) * HD;
                    mbar_wait(&qd_empty[s], ph ^ 1, 32);
                    mbar_expect_tx(&qd_full[s], 2 * QT_BYTES);
                    tma_load_chunked<HD, BWD_QT>(sQ + s * QT_BYTES, &tq64, &tqR, &qd_full[s], q_col,
                                                 loc.doc_start + qi * BWD_QT);
                    tma_load_chunked<HD, BWD_QT>(sO + s * QT_BYTES, &to64, &toR, &qd_full[s],
                                                 (group * p.q_per_group + hl) * HD, loc.doc_start + qi * BWD_QT);
                    if (++s == QDO_STAGES) s = 0, ph ^= 1;
                }
            }
        } else if (warp == 1) {
            int s = 0;
            uint32_t ph = 0;
            for (int n = 0; n < n_steps; ++n) {
                const int hl = n / n_i, qi = i0 + n % n_i;
                const int64_t row0 = int64_t(group * p.q_per_group + hl) * p.T + loc.doc_start;
                mbar_wait(&qd_empty[s], ph ^ 1, 33);
                float* ls = sL + s * 2 * BWD_QT;
#pragma unroll
                for (int r = lane; r < BWD_QT; r += 32) {
                    const int q = qi * BWD_QT + r;
                    ls[r] = q < loc.doc_len ? __ldg(p.lse + row0 + q) * log2e : 0.f;
                    ls[BWD_QT + r] = q < loc.doc_len ? __ldg(p.delta + row0 + q) : 0.f;
                }
                mbar_arrive(&qd_full[s]);
                if (++s == QDO_STAGES) s = 0, ph ^= 1;
            }
        }
        return;
    }

    // ================= consumers: warpgroup cw owns key rows [k0 + 64 cw, k0 + 64 cw + 64) =================
    setmaxnreg_inc<ATT_CONSUMER_REGS>();
    const int cw = wg - 1;
    const int n_steps_u = __shfl_sync(0xffffffffu, n_steps, 0);  // warp-uniform to ptxas, see attn_dq_kernel
    const int wr = (warp & 3) * 16 + (lane >> 2);  // first of the two accumulator rows of this thread (and wr + 8)
    const int wc = 2 * (lane & 3);                 // first accumulator column inside each n8 block
    const int kr[2] = {k0 + cw * 64 + wr, k0 + cw * 64 + wr + 8};  // doc-relative keys of the two rows
    const bool drop = p.drop.threshold != 0;
    const uint32_t sk0 = smem_u32(sK), sv0 = smem_u32(sV);

    float dv[HD / 2], dk[HD / 2];
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) dv[i] = dk[i] = 0.f;
    float st[BWD_QT / 2], dpt[BWD_QT / 2];

    // S^T, dP^T of the step in ring stage s (one commit group)
    auto issue_ss = [&](int s) {
        const uint32_t sq = smem_u32(sQ + s * QT_BYTES), so = smem_u32(sO + s * QT_BYTES);
        uint32_t sk = sk0, sv = sv0;
        opaque(sk), opaque(sv);
        wgmma_fence();
#pragma unroll
        for (int c = 0; c < CH::NCHUNK; ++c) {
            const int w = CH::width(c);
            const uint32_t krow = CH::offset(c, ATT_TILE) + cw * 64 * 2 * w;  // this warpgroup's 64 key rows of the chunk
#pragma unroll
            for (int k = 0; k < w / 16; ++k) {
                wgmma_ss<BWD_QT, 0, 0>(st, chunk_desc_kmajor(sk + krow, w, k), chunk_desc_kmajor(sq + CH::offset(c, BWD_QT), w, k),
                                       (c != 0 || k != 0) ? 1u : 0u);
                wgmma_ss<BWD_QT, 0, 0>(dpt, chunk_desc_kmajor(sv + krow, w, k), chunk_desc_kmajor(so + CH::offset(c, BWD_QT), w, k),
                                       (c != 0 || k != 0) ? 1u : 0u);
            }
        }
        wgmma_commit();
    };

    mbar_spin(kv_full, 0);
    int s = 0;
    uint32_t ph = 0;
    for (int n = 0; n < n_steps_u; ++n) {
        const int hl = n / n_i, qi = i0 + n % n_i;
        const int head = group * p.q_per_group + hl;
        const int q0 = qi * BWD_QT;
        const uint32_t head_key = dropout_head_key(uint32_t(head), p.drop.key0, p.drop.key1);
        mbar_spin(&qd_full[s], ph);
        issue_ss(s);
        wgmma_wait<0>();
        reg_fence<BWD_QT / 2>(st);
        reg_fence<BWD_QT / 2>(dpt);

        // ---------------- P^T, dS^T ----------------
        const float* ls = sL + s * 2 * BWD_QT;
        if (qi <= i0 + cw || (qi + 1) * BWD_QT > loc.doc_len)
            bwd_p_ds<ALIBI, true>(st, dpt, ls, ls + BWD_QT, p, loc, q0, wc, kr, head, head_key, drop);
        else
            bwd_p_ds<ALIBI, false>(st, dpt, ls, ls + BWD_QT, p, loc, q0, wc, kr, head, head_key, drop);
        uint32_t pa[BWD_QT / 16][4], da[BWD_QT / 16][4];
#pragma unroll
        for (int kk = 0; kk < BWD_QT / 16; ++kk) {
            acc_to_a_frag(st, kk, pa[kk]);
            acc_to_a_frag(dpt, kk, da[kk]);
        }

        // ---------------- dV += P^T dO,  dK += dS^T Q ----------------
        uint32_t sq = smem_u32(sQ + s * QT_BYTES), so = smem_u32(sO + s * QT_BYTES);
        opaque(sq), opaque(so);
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
        __syncwarp();
        mbar_arrive_lane0(&qd_empty[s], lane);  // Q_i / dO_i / LSE_i / Delta_i of this warp's step are read
        if (++s == QDO_STAGES) s = 0, ph ^= 1;
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

template <int HD, bool ALIBI>
int launch_bwd(const void* dout, const void* qkv, int64_t row_stride, const BwdParams& p, cudaStream_t st) {
    using CH = HeadChunks<HD>;
    CUtensorMap tq64, tqR, to64, toR;
    int rc = attn_make_maps<HD>(qkv, row_stride, p.T, &tq64, &tqR);
    if (rc) return rc;
    rc = attn_make_maps<HD>(dout, int64_t(p.n_heads) * HD, p.T, &to64, &toR);
    if (rc) return rc;
    constexpr int smem_bytes = 1024 + 2 * CH::tile_bytes(ATT_TILE) + 2 * QDO_STAGES * CH::tile_bytes(BWD_QT) +
                               QDO_STAGES * 2 * BWD_QT * 4 + 128;
    static_assert(smem_bytes <= 232448, "attention backward shared memory budget exceeded");
    auto kern = attn_bwd_kernel<HD, ALIBI>;
    static bool attr_set = false;
    if (!attr_set) {
        DOLO_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
        attr_set = true;
    }
    const int64_t max_tiles = (p.T + ATT_TILE - 1) / ATT_TILE + p.n_docs;
    DOLO_REQUIRE(max_tiles == p.n_tile_slots && max_tiles * p.n_groups < (1ll << 31), "attn_bwd: grid too large");
    dim3 grid((unsigned)(max_tiles * p.n_groups));
    kern<<<grid, ATT_BWD_THREADS, smem_bytes, st>>>(tq64, tqR, to64, toR, p);
    DOLO_LAUNCH_OK("attn_varlen_bwd");
    return DOLO_OK;
}

// dQ of the backward: one CTA = one 128-row query tile of one head of one document, two consumer warpgroups of 64 queries
// each, looping over the 64-row key tiles the queries see, in order.  Per key tile every consumer warpgroup recomputes
//     S  = Q_i K_j^T ,  dP = dO_i V_j^T           (SS)
//     dS = scale * P o (dP - Delta_i)             (registers, P = exp2(S*scale - LSE_i))
//     dQ_i += dS K_j                              (RS, B = K MN-major)
// and finally writes dQ_i (bf16) into the q slots of dqkv.  Thread 0 loads Q_i and dO_i once; an elected producer lane
// streams (K_j, V_j) through a KV_STAGES-deep ring.  Only the key tiles that reach the warpgroup's diagonal, and every key
// tile of a query tile that crosses the document end, test the causal / bounds predicate.  The SS MMAs of key tile j + 1
// are issued right behind the RS MMAs of key tile j.  ALIBI: P = exp2(log2(e) * (S*scale + bias_k) - LSE_i), one bias per
// key column of the thread.
constexpr int DQ_KT = 64;  // keys per step
constexpr int KV_STAGES = 4;

// dS (into sc) of key tile j from S, dP; MASK = test causality and the document end per element
template <bool ALIBI, bool MASK>
__device__ __forceinline__ void dq_ds(float (&sc)[DQ_KT / 2], const float (&dp)[DQ_KT / 2], const BwdParams& p,
                                      const TileLoc& loc, int j, int wc, const int (&qr)[2], const float (&lse_r)[2],
                                      const float (&del_r)[2], float slope, uint32_t head_key, bool drop) {
    if constexpr (ALIBI) {
#pragma unroll
        for (int b = 0; b < DQ_KT / 8; ++b)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int k = j * DQ_KT + 8 * b + wc + e;
                const float bl = attn_alibi_bias(slope, k) * ATT_LOG2E;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int i = 4 * b + 2 * h + e;
                    const bool ok = !MASK || (k <= qr[h] && qr[h] < loc.doc_len);
                    const float pr = ok ? fast_exp2(fmaf(sc[i], p.scale_log2, bl) - lse_r[h]) : 0.f;
                    float d = dp[i];
                    if (drop) d *= attn_drop_scale(p.drop, head_key, loc.doc_start + qr[h], loc.doc_start + k);
                    sc[i] = p.scale * pr * (d - del_r[h]);
                }
            }
    } else {
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int b = 0; b < DQ_KT / 8; ++b)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int k = j * DQ_KT + 8 * b + wc + e;
                    const int i = 4 * b + 2 * h + e;
                    const bool ok = !MASK || (k <= qr[h] && qr[h] < loc.doc_len);  // causal, and a real query of the document
                    const float pr = ok ? fast_exp2(fmaf(sc[i], p.scale_log2, -lse_r[h])) : 0.f;
                    float d = dp[i];
                    if (drop) d *= attn_drop_scale(p.drop, head_key, loc.doc_start + qr[h], loc.doc_start + k);
                    sc[i] = p.scale * pr * (d - del_r[h]);
                }
    }
}

template <int HD, bool ALIBI>
__global__ void __launch_bounds__(ATT_BWD_THREADS, 1)
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
    uint8_t* sO = sQ + Q_BYTES;               // dO
    uint8_t* sK = sO + Q_BYTES;               // [KV_STAGES]
    uint8_t* sV = sK + KV_STAGES * KT_BYTES;  // [KV_STAGES]
    uint64_t* bars = reinterpret_cast<uint64_t*>(sV + KV_STAGES * KT_BYTES);
    uint64_t* q_full = bars;                    // 1
    uint64_t* kv_full = bars + 1;               // [KV_STAGES]
    uint64_t* kv_empty = bars + 1 + KV_STAGES;  // [KV_STAGES], one arrive per consumer warp

    const int wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tq64);
        tma_prefetch_desc(&to64);
        if (CH::REM > 0) {
            tma_prefetch_desc(&tqR);
            tma_prefetch_desc(&toR);
        }
        mbar_init(q_full, 1);
        for (int i = 0; i < KV_STAGES; ++i) {
            mbar_init(&kv_full[i], 1);
            mbar_init(&kv_empty[i], 8);
        }
        mbar_fence_init();
        mbar_expect_tx(q_full, 2 * Q_BYTES);
        tma_load_chunked<HD, ATT_TILE>(sQ, &tq64, &tqR, q_full, q_col, loc.doc_start + q0);
        tma_load_chunked<HD, ATT_TILE>(sO, &to64, &toR, q_full, head * HD, loc.doc_start + q0);
    }
    __syncthreads();

    if (wg == 0) {
        // ================= producer =================
        setmaxnreg_dec<ATT_PRODUCER_REGS>();
        if (warp == 0 && elect_one()) {
            int s = 0;
            uint32_t ph = 0;
            for (int j = 0; j < n_kt; ++j) {
                mbar_wait(&kv_empty[s], ph ^ 1, 42);
                mbar_expect_tx(&kv_full[s], 2 * KT_BYTES);
                tma_load_chunked<HD, DQ_KT>(sK + s * KT_BYTES, &tq64, &tqR, &kv_full[s], k_col, loc.doc_start + j * DQ_KT);
                tma_load_chunked<HD, DQ_KT>(sV + s * KT_BYTES, &tq64, &tqR, &kv_full[s], v_col, loc.doc_start + j * DQ_KT);
                if (++s == KV_STAGES) s = 0, ph ^= 1;
            }
        }
        return;
    }

    // ================= consumers: warpgroup cw owns queries [q0 + 64 cw, q0 + 64 cw + 64) =================
    setmaxnreg_inc<ATT_CONSUMER_REGS>();
    const int cw = wg - 1;
    // the key-tile count, read back through a shuffle, is warp-uniform to ptxas: the loop branches with an SS group in flight
    const int n_kt_u = __shfl_sync(0xffffffffu, n_kt, 0);
    const int wr = (warp & 3) * 16 + (lane >> 2);
    const int wc = 2 * (lane & 3);
    const int qr[2] = {q0 + cw * 64 + wr, q0 + cw * 64 + wr + 8};  // doc-relative queries of the two rows
    const bool drop = p.drop.threshold != 0;
    const uint32_t head_key = dropout_head_key(uint32_t(head), p.drop.key0, p.drop.key1);
    const float log2e = 1.4426950408889634f;
    const float slope = ALIBI ? __ldg(p.alibi_slopes + head) : 0.f;
    float lse_r[2], del_r[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const bool ok = qr[h] < loc.doc_len;
        const int64_t idx = int64_t(head) * p.T + loc.doc_start + qr[h];
        lse_r[h] = ok ? __ldg(p.lse + idx) * log2e : 0.f;
        del_r[h] = ok ? __ldg(p.delta + idx) : 0.f;
    }
    // key tiles j >= j_diag reach this warpgroup's diagonal; all of them test the predicate if its rows cross the document end
    const int j_diag = (q0 + cw * 64 + 64 > loc.doc_len) ? 0 : q0 / DQ_KT + cw;
    const uint32_t sq = smem_u32(sQ), so = smem_u32(sO);
    float dq[HD / 2];
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) dq[i] = 0.f;
    float sc[DQ_KT / 2], dp[DQ_KT / 2];

    // S, dP of the key tile in ring stage s (one commit group)
    auto issue_ss = [&](int s) {
        uint32_t sk = smem_u32(sK + s * KT_BYTES), sv = smem_u32(sV + s * KT_BYTES);
        opaque(sk), opaque(sv);
        wgmma_fence();
#pragma unroll
        for (int c = 0; c < CH::NCHUNK; ++c) {
            const int w = CH::width(c);
            const uint32_t qrow = CH::offset(c, ATT_TILE) + cw * 64 * 2 * w;  // this warpgroup's 64 query rows of the chunk
#pragma unroll
            for (int k = 0; k < w / 16; ++k) {
                wgmma_ss<DQ_KT, 0, 0>(sc, chunk_desc_kmajor(sq + qrow, w, k), chunk_desc_kmajor(sk + CH::offset(c, DQ_KT), w, k),
                                      (c != 0 || k != 0) ? 1u : 0u);
                wgmma_ss<DQ_KT, 0, 0>(dp, chunk_desc_kmajor(so + qrow, w, k), chunk_desc_kmajor(sv + CH::offset(c, DQ_KT), w, k),
                                      (c != 0 || k != 0) ? 1u : 0u);
            }
        }
        wgmma_commit();
    };

    mbar_spin(q_full, 0);
    int s = 0;
    uint32_t ph = 0;
    mbar_spin(&kv_full[0], 0);
    issue_ss(0);
    for (int j = 0; j < n_kt_u; ++j) {
        wgmma_wait<0>();
        reg_fence<DQ_KT / 2>(sc);
        reg_fence<DQ_KT / 2>(dp);
        if (j >= j_diag)
            dq_ds<ALIBI, true>(sc, dp, p, loc, j, wc, qr, lse_r, del_r, slope, head_key, drop);
        else
            dq_ds<ALIBI, false>(sc, dp, p, loc, j, wc, qr, lse_r, del_r, slope, head_key, drop);
        uint32_t da[DQ_KT / 16][4];
#pragma unroll
        for (int kk = 0; kk < DQ_KT / 16; ++kk) acc_to_a_frag(sc, kk, da[kk]);

        const int s1 = s + 1 == KV_STAGES ? 0 : s + 1;
        const uint32_t ph1 = s1 == 0 ? ph ^ 1 : ph;
        const bool more = j + 1 < n_kt_u;
        if (more) mbar_spin(&kv_full[s1], ph1);
        uint32_t sk = smem_u32(sK + s * KT_BYTES);
        opaque(sk);
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

        if (more) {
            issue_ss(s1);
            wgmma_wait<1>();  // the RS group of key tile j is done; the SS group of key tile j + 1 runs on
        } else {
            wgmma_wait<0>();
        }
        reg_fence<HD / 2>(dq);
        __syncwarp();
        mbar_arrive_lane0(&kv_empty[s], lane);  // K_j / V_j of this warp's MMAs are read
        s = s1, ph = ph1;
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

template <int HD, bool ALIBI>
int launch_dq(const void* dout, const void* qkv, int64_t row_stride, const BwdParams& p, cudaStream_t st) {
    using CH = HeadChunks<HD>;
    CUtensorMap tq64, tqR, to64, toR;
    int rc = attn_make_maps<HD>(qkv, row_stride, p.T, &tq64, &tqR);
    if (rc) return rc;
    rc = attn_make_maps<HD>(dout, int64_t(p.n_heads) * HD, p.T, &to64, &toR);
    if (rc) return rc;
    constexpr int smem_bytes = 1024 + 2 * CH::tile_bytes(ATT_TILE) + 2 * KV_STAGES * CH::tile_bytes(DQ_KT) + 128;
    static_assert(smem_bytes <= 232448, "attention dQ shared memory budget exceeded");
    auto kern = attn_dq_kernel<HD, ALIBI>;
    static bool attr_set = false;
    if (!attr_set) {
        DOLO_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
        attr_set = true;
    }
    const int64_t max_tiles = (p.T + ATT_TILE - 1) / ATT_TILE + p.n_docs;
    DOLO_REQUIRE(max_tiles == p.n_tile_slots && max_tiles * p.n_heads < (1ll << 31), "attn_bwd: grid too large");
    dim3 grid((unsigned)(max_tiles * p.n_heads));
    kern<<<grid, ATT_BWD_THREADS, smem_bytes, st>>>(tq64, tqR, to64, toR, p);
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

namespace {

template <int HD>
int launch_bwd_dq(const void* dout, const void* qkv, int64_t row_stride, const BwdParams& p, cudaStream_t st) {
    int rc;
    if (p.alibi_slopes != nullptr) {
        rc = launch_bwd<HD, true>(dout, qkv, row_stride, p, st);
        return rc ? rc : launch_dq<HD, true>(dout, qkv, row_stride, p, st);
    }
    rc = launch_bwd<HD, false>(dout, qkv, row_stride, p, st);
    return rc ? rc : launch_dq<HD, false>(dout, qkv, row_stride, p, st);
}

// alibi_slopes == nullptr: the plain kernels
int attn_bwd(const void* dout, const void* qkv, int64_t row_stride, const void* out, const float* lse, void* dqkv,
             const int32_t* cu_seqlens, int n_docs, int64_t T, int n_groups, int q_per_group, int head_dim,
             float softmax_scale, float dropout_p, uint32_t key0, uint32_t key1, const float* alibi_slopes, void* workspace,
             void* stream) {
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
    switch (head_dim) {
        case 16: case 32: case 64: case 80: case 96: case 128: case 160: case 192: case 256: break;
        default: return dolo_set_error("attn_bwd: unsupported head_dim %d (supported: 16,32,64,80,96,128,160,192,256)", head_dim);
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    float* delta = static_cast<float*>(workspace);
    {
        const int64_t blocks = (T + DELTA_TOK - 1) / DELTA_TOK;
        attn_delta_kernel<<<(unsigned)blocks, 256, size_t(nh) * (head_dim / 8) * DELTA_TOK * sizeof(float), st>>>(
            static_cast<const uint4*>(dout), static_cast<const uint4*>(out), delta, T, nh, head_dim / 8);
        DOLO_LAUNCH_OK("attn_delta");
    }
    if (head_dim > 128)
        return dolo_attn_wide_bwd(dout, qkv, row_stride, lse, delta, dqkv, cu_seqlens, n_docs, T, n_groups, q_per_group,
                                  head_dim, softmax_scale, dropout_p, key0, key1, alibi_slopes, st);
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
    p.alibi_slopes = alibi_slopes;
    switch (head_dim) {
        case 16: return launch_bwd_dq<16>(dout, qkv, row_stride, p, st);
        case 32: return launch_bwd_dq<32>(dout, qkv, row_stride, p, st);
        case 64: return launch_bwd_dq<64>(dout, qkv, row_stride, p, st);
        case 80: return launch_bwd_dq<80>(dout, qkv, row_stride, p, st);
        case 96: return launch_bwd_dq<96>(dout, qkv, row_stride, p, st);
        default: return launch_bwd_dq<128>(dout, qkv, row_stride, p, st);
    }
}

}  // namespace

extern "C" int dolomite_b200_attn_varlen_bwd_dropout(const void* dout, const void* qkv, int64_t row_stride, const void* out,
                                                     const float* lse, void* dqkv, const int32_t* cu_seqlens, int n_docs,
                                                     int64_t T, int max_seqlen, int n_groups, int q_per_group,
                                                     int head_dim, float softmax_scale, float dropout_p, uint32_t key0,
                                                     uint32_t key1, void* workspace, void* stream) {
    (void)max_seqlen;
    return attn_bwd(dout, qkv, row_stride, out, lse, dqkv, cu_seqlens, n_docs, T, n_groups, q_per_group, head_dim,
                    softmax_scale, dropout_p, key0, key1, nullptr, workspace, stream);
}

extern "C" int dolomite_b200_attn_varlen_bwd_alibi(const void* dout, const void* qkv, int64_t row_stride, const void* out,
                                                   const float* lse, void* dqkv, const int32_t* cu_seqlens, int n_docs,
                                                   int64_t T, int max_seqlen, int n_groups, int q_per_group, int head_dim,
                                                   float softmax_scale, float dropout_p, uint32_t key0, uint32_t key1,
                                                   const float* alibi_slopes, void* workspace, void* stream) {
    (void)max_seqlen;
    DOLO_REQUIRE(alibi_slopes != nullptr, "attn_bwd_alibi: alibi_slopes is null");
    return attn_bwd(dout, qkv, row_stride, out, lse, dqkv, cu_seqlens, n_docs, T, n_groups, q_per_group, head_dim,
                    softmax_scale, dropout_p, key0, key1, alibi_slopes, workspace, stream);
}
