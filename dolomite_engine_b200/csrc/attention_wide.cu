// Packed var-len causal attention for wide heads (head_dim 160, 192, 256) on wgmma: forward, backward (dK / dV and dQ) and
// decode.  Each kernel computes what its narrow counterpart (attention_fwd.cu, attention_bwd.cu, attention_decode.cu)
// computes -- qkv slot layout, per-document causal mask, natural-log LSE, dropout keys, ALiBi bias, KV-cache layout, dK / dV
// summed over the q heads of a group in a fixed order -- with tiles that fit at head_dim 256, where the narrow tiling does
// not: its forward would hold 64 + 32 + 16 fp32 / packed values per thread on top of o[128], its shared memory would exceed
// 227 KB, and its dK / dV warpgroup would hold 2 x 128 accumulators.
//
//   forward  128-query tile, two warpgroups of 64 rows, 64-key K / V tiles through a 2-stage ring
//   dK / dV  64 key rows per CTA (half of a 128-key tile): warpgroup A runs S^T = K Q^T, P^T and dV += P^T dO, warpgroup B
//            runs dP^T = V dO^T, dS^T and dK += dS^T Q; A hands the fp32 P^T to B through shared memory, in fragment order
//   dQ       64 query rows per CTA (half of a 128-query tile), 64-key tiles in order through a 2-stage ring
//   decode   one CTA per (sequence, head), 256 threads, one output column per thread
//
// head_dim 160 = 64 + 64 + 32; 192 and 256 are whole 64-column chunks (HeadChunks).
#include "attention_common.cuh"
#include "../../include/dolomite_b200.h"

using namespace dolo;

uint32_t dolo_dropout_threshold(float p);  // dropout.cu

namespace {

constexpr int WIDE_KT = 64;     // keys per K / V tile (forward, dQ); query rows per step and key rows per CTA (dK / dV)
constexpr int WIDE_STAGES = 2;  // depth of every ring

struct WideParams {
    const int32_t* cu_seqlens;
    int n_docs;
    int64_t T;
    int n_groups, q_per_group, n_heads;
    float scale, scale_log2;
    AttnDropout drop;           // threshold 0: none
    int head_chunk;             // CTA order (attn_cta_order): heads (forward, dQ) or kv groups (dK / dV) per chunk
    int n_slots;                // tile slots per head of the grid: 128-row tiles (forward), 64-row halves (backward)
    const float* alibi_slopes;  // [n_heads] fp32, read by the ALIBI instances only
    __nv_bfloat16* out;         // forward: [T, n_heads * HD]
    float* lse_out;             // forward: [n_heads, T]
    const float* lse;           // backward: [n_heads, T]
    const float* delta;         // backward: [n_heads, T]
    __nv_bfloat16* dqkv;        // backward: [T, row_stride]
    int64_t row_stride;
};

// ================================================================================================================
// forward
// ================================================================================================================
// One CTA = one 128-row query tile of one head of one document, two warpgroups of 64 query rows; thread 0 also issues the
// TMA loads (Q once, then (K_j, V_j) of 64 keys through the ring).  Warpgroup w walks key tiles 0 .. j_diag(w), the last
// one holding its diagonal; a warpgroup whose rows all lie past the document end computes nothing.  Per key tile:
//     S = Q K_j^T (SS, 64 x 64 fp32)   online softmax   O += P V_j (RS)
// exactly as attn_fwd_kernel, and the same epilogue.  Per thread at head_dim 256: o 128 + S 32 + P fragments 16.
constexpr int WFWD_THREADS = 256;

template <int HD, bool ALIBI>
__global__ void __launch_bounds__(WFWD_THREADS, 1)
    attn_wide_fwd_kernel(const __grid_constant__ CUtensorMap tmap64, const __grid_constant__ CUtensorMap tmapR,
                         const WideParams p) {
    using CH = HeadChunks<HD>;
    constexpr int Q_BYTES = CH::tile_bytes(ATT_TILE);
    constexpr int KT_BYTES = CH::tile_bytes(WIDE_KT);

    int ti, head;
    attn_cta_order(p.head_chunk, p.n_slots, ti, head);
    ti = p.n_slots - 1 - ti;  // long (late) tiles first
    const TileLoc loc = locate_tile(p.cu_seqlens, p.n_docs, ti);
    if (!loc.valid) return;  // uniform for the whole CTA
    const int group = head / p.q_per_group, slot = head % p.q_per_group;
    const int q_col = (group * (p.q_per_group + 2) + slot) * HD;
    const int k_col = (group * (p.q_per_group + 2) + p.q_per_group) * HD;
    const int v_col = k_col + HD;
    const int q0 = loc.tile * ATT_TILE;
    const int n_kt = (min(q0 + ATT_TILE, loc.doc_len) + WIDE_KT - 1) / WIDE_KT;  // key tiles some query of the tile sees

    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_align_1024(smem_raw);
    uint8_t* sQ = smem;
    uint8_t* sK = sQ + Q_BYTES;                 // [WIDE_STAGES]
    uint8_t* sV = sK + WIDE_STAGES * KT_BYTES;  // [WIDE_STAGES]
    uint64_t* bars = reinterpret_cast<uint64_t*>(sV + WIDE_STAGES * KT_BYTES);
    uint64_t* q_full = bars;                       // 1
    uint64_t* kv_full = bars + 1;                  // [WIDE_STAGES]
    uint64_t* kv_empty = bars + 1 + WIDE_STAGES;   // [WIDE_STAGES], one arrive per warp

    const int wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    auto load_kv = [&](int j, int s) {
        mbar_expect_tx(&kv_full[s], 2 * KT_BYTES);
        tma_load_chunked<HD, WIDE_KT>(sK + s * KT_BYTES, &tmap64, &tmapR, &kv_full[s], k_col, loc.doc_start + j * WIDE_KT);
        tma_load_chunked<HD, WIDE_KT>(sV + s * KT_BYTES, &tmap64, &tmapR, &kv_full[s], v_col, loc.doc_start + j * WIDE_KT);
    };
    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmap64);
        if (CH::REM > 0) tma_prefetch_desc(&tmapR);
        mbar_init(q_full, 1);
        for (int i = 0; i < WIDE_STAGES; ++i) {
            mbar_init(&kv_full[i], 1);
            mbar_init(&kv_empty[i], WFWD_THREADS / 32);
        }
        mbar_fence_init();
        mbar_expect_tx(q_full, Q_BYTES);
        tma_load_chunked<HD, ATT_TILE>(sQ, &tmap64, &tmapR, q_full, q_col, loc.doc_start + q0);
        for (int j = 0; j < WIDE_STAGES && j < n_kt; ++j) load_kv(j, j);
    }
    __syncthreads();

    const int wr = (warp & 3) * 16 + (lane >> 2);  // first of the two accumulator rows of this thread (and wr + 8)
    const int wc = 2 * (lane & 3);                 // first accumulator column inside each n8 block
    const int qw = q0 + wg * 64;                   // first query (doc-relative) of this warpgroup
    const int qr[2] = {qw + wr, qw + wr + 8};
    const int j_diag = qw / WIDE_KT;                                 // the key tile of this warpgroup's diagonal
    const int n_kt_wg = qw < loc.doc_len ? j_diag + 1 : 0;           // <= n_kt
    const bool drop = p.drop.threshold != 0;
    const uint32_t head_key = dropout_head_key(uint32_t(head), p.drop.key0, p.drop.key1);
    const uint32_t sq = smem_u32(sQ);

    float o[HD / 2];
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
    // row max (raw score; ALIBI: log2 units of the biased logit), thread-partial row sum
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    const float slope = ALIBI ? __ldg(p.alibi_slopes + head) : 0.f;

    mbar_wait(q_full, 0, 60);
    for (int j = 0; j < n_kt; ++j) {
        const int s = j & (WIDE_STAGES - 1);
        // every warpgroup waits for every tile, also one it skips: an arrive on kv_empty before the tile is loaded would
        // count towards a later phase of the ring barrier, and thread 0 would then wait on a phase that never completes
        mbar_wait(&kv_full[s], (j / WIDE_STAGES) & 1, 61);
        if (j < n_kt_wg) {  // warpgroup-uniform; once false it stays false
            const uint32_t sk = smem_u32(sK + s * KT_BYTES), sv = smem_u32(sV + s * KT_BYTES);
            float sc[WIDE_KT / 2];
            wgmma_fence();
#pragma unroll
            for (int c = 0; c < CH::NCHUNK; ++c) {
                const int w = CH::width(c);
#pragma unroll
                for (int k = 0; k < w / 16; ++k)
                    wgmma_ss<WIDE_KT, 0, 0>(sc, chunk_desc_kmajor(sq + CH::offset(c, ATT_TILE) + wg * 64 * 2 * w, w, k),
                                            chunk_desc_kmajor(sk + CH::offset(c, WIDE_KT), w, k), (c != 0 || k != 0) ? 1u : 0u);
            }
            wgmma_commit();
            wgmma_wait<0>();
            reg_fence<WIDE_KT / 2>(sc);

            // ---------------- online softmax over this key tile ----------------
            const bool diag = j == j_diag;  // only the diagonal tile has keys past a query of the warpgroup
            const int kbase = j * WIDE_KT + wc;
            if constexpr (ALIBI) {  // sc <- log2(e) * (scale * s + bias_k)
#pragma unroll
                for (int b = 0; b < WIDE_KT / 8; ++b)
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
                for (int b = 0; b < WIDE_KT / 8; ++b)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        float& x = sc[4 * b + 2 * h + e];
                        if (diag && kbase + 8 * b + e > qr[h]) x = -INFINITY;
                        mx = fmaxf(mx, x);
                    }
                mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
                mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
                // key 0 precedes every query: the row max is finite from key tile 0 on
                const float corr = ALIBI ? fast_exp2(m_run[h] - mx) : fast_exp2((m_run[h] - mx) * p.scale_log2);
                const float neg_m = ALIBI ? -mx : -mx * p.scale_log2;
                float lsum = 0.f;
#pragma unroll
                for (int b = 0; b < WIDE_KT / 8; ++b)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        float& x = sc[4 * b + 2 * h + e];
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
            uint32_t pa[WIDE_KT / 16][4];
#pragma unroll
            for (int kk = 0; kk < WIDE_KT / 16; ++kk) acc_to_a_frag(sc, kk, pa[kk]);

            // ---------------- O += P V_j ----------------
            wgmma_fence();
#pragma unroll
            for (int c = 0; c < CH::NCHUNK; ++c) {
#pragma unroll
                for (int kk = 0; kk < WIDE_KT / 16; ++kk) {
                    if (CH::width(c) == 64)
                        wgmma_rs<64, 1>(o + CH::col(c) / 2, pa[kk], chunk_desc_mnmajor(sv + CH::offset(c, WIDE_KT), 64, kk), 1u);
                    else
                        wgmma_rs<(CH::REM ? CH::REM : 16), 1>(o + CH::col(c) / 2, pa[kk],
                                                              chunk_desc_mnmajor(sv + CH::offset(c, WIDE_KT), CH::REM, kk), 1u);
                }
            }
            wgmma_commit();
            wgmma_wait<0>();
            reg_fence<HD / 2>(o);
        }
        if (lane == 0) mbar_arrive(&kv_empty[s]);
        if (threadIdx.x == 0 && j + WIDE_STAGES < n_kt) {
            mbar_wait(&kv_empty[s], (j / WIDE_STAGES) & 1, 62);  // both warpgroups are done with tile j
            load_kv(j + WIDE_STAGES, s);
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
            p.lse_out[int64_t(head) * p.T + row] = (ALIBI ? m_run[h] * ATT_LN2 : m_run[h] * p.scale) + logf(l);
    }
}

template <int HD, bool ALIBI>
int launch_wide_fwd(const void* qkv, int64_t row_stride, const WideParams& p, cudaStream_t st) {
    using CH = HeadChunks<HD>;
    CUtensorMap t64, tR;
    int rc = attn_make_maps<HD>(qkv, row_stride, p.T, &t64, &tR);
    if (rc) return rc;
    constexpr int smem_bytes = 1024 + CH::tile_bytes(ATT_TILE) + 2 * WIDE_STAGES * CH::tile_bytes(WIDE_KT) + 128;
    static_assert(smem_bytes <= 232448, "wide attention forward shared memory budget exceeded");
    auto kern = attn_wide_fwd_kernel<HD, ALIBI>;
    static bool attr_set = false;
    if (!attr_set) {
        DOLO_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
        attr_set = true;
    }
    DOLO_REQUIRE(int64_t(p.n_slots) * p.n_heads < (1ll << 31), "attn_fwd: grid too large");
    kern<<<dim3(unsigned(p.n_slots * p.n_heads)), WFWD_THREADS, smem_bytes, st>>>(t64, tR, p);
    DOLO_LAUNCH_OK("attn_varlen_fwd");
    return DOLO_OK;
}

// ================================================================================================================
// backward: dK / dV
// ================================================================================================================
// One CTA = 64 key rows (one half of a 128-key tile) of one kv group of one document; it loops over the q heads of the
// group and the 64-row query tiles that see its keys, as attn_bwd_kernel does, in the same "transposed" frame (accumulator
// row == key row).  Warpgroup 0 is the producer (thread 0 loads K, V once; an elected lane of warp 0 streams Q_i, dO_i
// through the ring; warp 1 stages LSE_i * log2 e and Delta_i).  The two consumer warpgroups split the outputs, so that each
// holds one 64 x HD accumulator and runs two MMAs per step:
//     A (warpgroup 1):  S^T = K Q_i^T (SS)   P^T = exp2(S^T*scale - LSE_i)   dV += (Z o P^T) dO_i (RS)
//     B (warpgroup 2):  dP^T = V dO_i^T (SS)   dS^T = scale * P^T o (Z o dP^T - Delta_i)   dK += dS^T Q_i (RS)
// A writes its fp32 P^T (before dropout) to shared memory in fragment order -- element i of thread t at [i][t], so every
// store and load of a warp is one conflict-free row -- and signals B on named barrier PT_FULL; B signals that it has read it
// on PT_FREE.  No wgmma group is in flight at either barrier.  Per thread at head_dim 256: 128 + 32 + 16 in each warpgroup.
constexpr int WBWD_THREADS = 384;
constexpr int WIDE_PRODUCER_REGS = 24;
constexpr int WIDE_CONSUMER_REGS = 240;
static_assert(WIDE_PRODUCER_REGS * 128 + 2 * WIDE_CONSUMER_REGS * 128 <= 65536, "register file exceeded");
constexpr uint32_t BAR_PT_FULL = 1, BAR_PT_FREE = 2;  // named barriers of warpgroups A and B (256 threads)

// P^T of one step into sPt (undropped) and st (dropped and rescaled: what dV sees); MASK = test causality and the document
// end per element
template <bool ALIBI, bool MASK>
__device__ __forceinline__ void wide_pt(float (&st)[WIDE_KT / 2], float* sPt, const float* ls, const WideParams& p,
                                        const TileLoc& loc, int q0, int wc, const int (&kr)[2], float slope,
                                        uint32_t head_key, bool drop) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const float bias_r = ALIBI ? attn_alibi_bias(slope, kr[h]) * ATT_LOG2E : 0.f;  // log2(e) * bias of the key row
#pragma unroll
        for (int b = 0; b < WIDE_KT / 8; ++b) {
            const float2 l = *reinterpret_cast<const float2*>(ls + 8 * b + wc);
            const float lse_c[2] = {l.x, l.y};
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
                sPt[i * 128] = pr;
                st[i] = drop ? pr * attn_drop_scale(p.drop, head_key, loc.doc_start + q, loc.doc_start + kr[h]) : pr;
            }
        }
    }
}

template <int HD, bool ALIBI>
__global__ void __launch_bounds__(WBWD_THREADS, 1)
    attn_wide_bwd_kernel(const __grid_constant__ CUtensorMap tq64, const __grid_constant__ CUtensorMap tqR,
                         const __grid_constant__ CUtensorMap to64, const __grid_constant__ CUtensorMap toR,
                         const WideParams p) {
    using CH = HeadChunks<HD>;
    constexpr int T_BYTES = CH::tile_bytes(WIDE_KT);  // K, V, and a Q_i / dO_i step: 64 rows each

    int half, group;  // 64-row halves of the 128-key tiles in natural order = longest first
    attn_cta_order(p.head_chunk, p.n_slots, half, group);
    const TileLoc loc = locate_tile(p.cu_seqlens, p.n_docs, half >> 1);
    if (!loc.valid) return;
    const int k0 = loc.tile * ATT_TILE + (half & 1) * WIDE_KT;  // first key (doc-relative) of this CTA
    if (k0 >= loc.doc_len) return;
    const int i0 = k0 / WIDE_KT;  // first (diagonal) query tile
    const int n_i = (loc.doc_len + WIDE_KT - 1) / WIDE_KT - i0;
    const int n_steps = n_i * p.q_per_group;
    const int k_col = (group * (p.q_per_group + 2) + p.q_per_group) * HD;
    const int v_col = k_col + HD;

    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_align_1024(smem_raw);
    uint8_t* sK = smem;
    uint8_t* sV = sK + T_BYTES;
    uint8_t* sQ = sV + T_BYTES;                   // [WIDE_STAGES]
    uint8_t* sO = sQ + WIDE_STAGES * T_BYTES;     // [WIDE_STAGES] dO
    float* sP = reinterpret_cast<float*>(sO + WIDE_STAGES * T_BYTES);  // [32][128] P^T of one step, fragment order
    float* sL = sP + WIDE_KT * WIDE_KT;           // [WIDE_STAGES][LSE * log2 e, Delta][WIDE_KT]
    uint64_t* bars = reinterpret_cast<uint64_t*>(sL + WIDE_STAGES * 2 * WIDE_KT);
    uint64_t* kv_full = bars;                      // 1
    uint64_t* qd_full = bars + 1;                  // [WIDE_STAGES]: TMA bytes + one arrive per lane of producer warp 1
    uint64_t* qd_empty = bars + 1 + WIDE_STAGES;   // [WIDE_STAGES], one arrive per consumer warp

    const int wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tq64);
        tma_prefetch_desc(&to64);
        if (CH::REM > 0) {
            tma_prefetch_desc(&tqR);
            tma_prefetch_desc(&toR);
        }
        mbar_init(kv_full, 1);
        for (int i = 0; i < WIDE_STAGES; ++i) {
            mbar_init(&qd_full[i], 1 + 32);
            mbar_init(&qd_empty[i], 8);
        }
        mbar_fence_init();
        mbar_expect_tx(kv_full, 2 * T_BYTES);
        tma_load_chunked<HD, WIDE_KT>(sK, &tq64, &tqR, kv_full, k_col, loc.doc_start + k0);
        tma_load_chunked<HD, WIDE_KT>(sV, &tq64, &tqR, kv_full, v_col, loc.doc_start + k0);
    }
    __syncthreads();

    if (wg == 0) {
        // ================= producer =================
        setmaxnreg_dec<WIDE_PRODUCER_REGS>();
        if (warp == 0) {
            if (elect_one()) {
                int s = 0;
                uint32_t ph = 0;
                for (int n = 0; n < n_steps; ++n) {
                    const int hl = n / n_i, qi = i0 + n % n_i;
                    const int q_col = (group * (p.q_per_group + 2) + hl) * HD;
                    mbar_wait(&qd_empty[s], ph ^ 1, 63);
                    mbar_expect_tx(&qd_full[s], 2 * T_BYTES);
                    tma_load_chunked<HD, WIDE_KT>(sQ + s * T_BYTES, &tq64, &tqR, &qd_full[s], q_col, loc.doc_start + qi * WIDE_KT);
                    tma_load_chunked<HD, WIDE_KT>(sO + s * T_BYTES, &to64, &toR, &qd_full[s], (group * p.q_per_group + hl) * HD,
                                                  loc.doc_start + qi * WIDE_KT);
                    if (++s == WIDE_STAGES) s = 0, ph ^= 1;
                }
            }
        } else if (warp == 1) {
            int s = 0;
            uint32_t ph = 0;
            for (int n = 0; n < n_steps; ++n) {
                const int hl = n / n_i, qi = i0 + n % n_i;
                const int64_t row0 = int64_t(group * p.q_per_group + hl) * p.T + loc.doc_start;
                mbar_wait(&qd_empty[s], ph ^ 1, 64);
                float* ls = sL + s * 2 * WIDE_KT;
#pragma unroll
                for (int r = lane; r < WIDE_KT; r += 32) {
                    const int q = qi * WIDE_KT + r;
                    ls[r] = q < loc.doc_len ? __ldg(p.lse + row0 + q) * ATT_LOG2E : 0.f;
                    ls[WIDE_KT + r] = q < loc.doc_len ? __ldg(p.delta + row0 + q) : 0.f;
                }
                mbar_arrive(&qd_full[s]);
                if (++s == WIDE_STAGES) s = 0, ph ^= 1;
            }
        }
        return;
    }

    // ================= consumers: both own key rows [k0, k0 + 64) =================
    setmaxnreg_inc<WIDE_CONSUMER_REGS>();
    const int n_steps_u = __shfl_sync(0xffffffffu, n_steps, 0);  // warp-uniform to ptxas, see attn_dq_kernel
    const int wr = (warp & 3) * 16 + (lane >> 2);
    const int wc = 2 * (lane & 3);
    const int kr[2] = {k0 + wr, k0 + wr + 8};  // doc-relative keys of the two rows
    const bool drop = p.drop.threshold != 0;
    float* sPt = sP + (threadIdx.x & 127);  // this thread's P^T elements, stride 128
    float acc[HD / 2];                      // A: dV, B: dK
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) acc[i] = 0.f;
    float sc[WIDE_KT / 2];                  // A: S^T, B: dP^T

    mbar_spin(kv_full, 0);
    int s = 0;
    uint32_t ph = 0;
    if (wg == 1) {
        // ---------------- A: S^T, P^T, dV ----------------
        for (int n = 0; n < n_steps_u; ++n) {
            const int hl = n / n_i, qi = i0 + n % n_i;
            const int head = group * p.q_per_group + hl;
            const int q0 = qi * WIDE_KT;
            const uint32_t head_key = dropout_head_key(uint32_t(head), p.drop.key0, p.drop.key1);
            const float slope = ALIBI ? __ldg(p.alibi_slopes + head) : 0.f;
            mbar_spin(&qd_full[s], ph);
            uint32_t sk = smem_u32(sK), sq = smem_u32(sQ + s * T_BYTES);
            opaque(sk), opaque(sq);
            wgmma_fence();
#pragma unroll
            for (int c = 0; c < CH::NCHUNK; ++c) {
                const int w = CH::width(c);
#pragma unroll
                for (int k = 0; k < w / 16; ++k)
                    wgmma_ss<WIDE_KT, 0, 0>(sc, chunk_desc_kmajor(sk + CH::offset(c, WIDE_KT), w, k),
                                            chunk_desc_kmajor(sq + CH::offset(c, WIDE_KT), w, k), (c != 0 || k != 0) ? 1u : 0u);
            }
            wgmma_commit();
            wgmma_wait<0>();
            reg_fence<WIDE_KT / 2>(sc);

            if (n > 0) named_bar_sync(BAR_PT_FREE, 256);  // B has read the P^T of the previous step
            const float* ls = sL + s * 2 * WIDE_KT;
            if (qi == i0 || (qi + 1) * WIDE_KT > loc.doc_len)
                wide_pt<ALIBI, true>(sc, sPt, ls, p, loc, q0, wc, kr, slope, head_key, drop);
            else
                wide_pt<ALIBI, false>(sc, sPt, ls, p, loc, q0, wc, kr, slope, head_key, drop);
            named_bar_arrive(BAR_PT_FULL, 256);
            uint32_t pa[WIDE_KT / 16][4];
#pragma unroll
            for (int kk = 0; kk < WIDE_KT / 16; ++kk) acc_to_a_frag(sc, kk, pa[kk]);

            uint32_t so = smem_u32(sO + s * T_BYTES);
            opaque(so);
            wgmma_fence();
#pragma unroll
            for (int c = 0; c < CH::NCHUNK; ++c) {
#pragma unroll
                for (int kk = 0; kk < WIDE_KT / 16; ++kk) {
                    if (CH::width(c) == 64) {
                        wgmma_rs<64, 1>(acc + CH::col(c) / 2, pa[kk], chunk_desc_mnmajor(so + CH::offset(c, WIDE_KT), 64, kk), 1u);
                    } else {
                        constexpr int R = CH::REM ? CH::REM : 16;
                        wgmma_rs<R, 1>(acc + CH::col(c) / 2, pa[kk], chunk_desc_mnmajor(so + CH::offset(c, WIDE_KT), R, kk), 1u);
                    }
                }
            }
            wgmma_commit();
            wgmma_wait<0>();
            reg_fence<HD / 2>(acc);
            __syncwarp();
            mbar_arrive_lane0(&qd_empty[s], lane);
            if (++s == WIDE_STAGES) s = 0, ph ^= 1;
        }
    } else {
        // ---------------- B: dP^T, dS^T, dK ----------------
        for (int n = 0; n < n_steps_u; ++n) {
            const int hl = n / n_i, qi = i0 + n % n_i;
            const int head = group * p.q_per_group + hl;
            const int q0 = qi * WIDE_KT;
            const uint32_t head_key = dropout_head_key(uint32_t(head), p.drop.key0, p.drop.key1);
            mbar_spin(&qd_full[s], ph);
            uint32_t sv = smem_u32(sV), so = smem_u32(sO + s * T_BYTES);
            opaque(sv), opaque(so);
            wgmma_fence();
#pragma unroll
            for (int c = 0; c < CH::NCHUNK; ++c) {
                const int w = CH::width(c);
#pragma unroll
                for (int k = 0; k < w / 16; ++k)
                    wgmma_ss<WIDE_KT, 0, 0>(sc, chunk_desc_kmajor(sv + CH::offset(c, WIDE_KT), w, k),
                                            chunk_desc_kmajor(so + CH::offset(c, WIDE_KT), w, k), (c != 0 || k != 0) ? 1u : 0u);
            }
            wgmma_commit();
            wgmma_wait<0>();
            reg_fence<WIDE_KT / 2>(sc);

            named_bar_sync(BAR_PT_FULL, 256);  // A's P^T of this step is in sP
            const float* ds = sL + s * 2 * WIDE_KT + WIDE_KT;
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int b = 0; b < WIDE_KT / 8; ++b) {
                    const float2 d = *reinterpret_cast<const float2*>(ds + 8 * b + wc);
                    const float del_c[2] = {d.x, d.y};
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int i = 4 * b + 2 * h + e;
                        float dp = sc[i];
                        if (drop)
                            dp *= attn_drop_scale(p.drop, head_key, loc.doc_start + q0 + 8 * b + wc + e, loc.doc_start + kr[h]);
                        sc[i] = p.scale * sPt[i * 128] * (dp - del_c[e]);
                    }
                }
            if (n + 1 < n_steps_u) named_bar_arrive(BAR_PT_FREE, 256);
            uint32_t da[WIDE_KT / 16][4];
#pragma unroll
            for (int kk = 0; kk < WIDE_KT / 16; ++kk) acc_to_a_frag(sc, kk, da[kk]);

            uint32_t sq = smem_u32(sQ + s * T_BYTES);
            opaque(sq);
            wgmma_fence();
#pragma unroll
            for (int c = 0; c < CH::NCHUNK; ++c) {
#pragma unroll
                for (int kk = 0; kk < WIDE_KT / 16; ++kk) {
                    if (CH::width(c) == 64) {
                        wgmma_rs<64, 1>(acc + CH::col(c) / 2, da[kk], chunk_desc_mnmajor(sq + CH::offset(c, WIDE_KT), 64, kk), 1u);
                    } else {
                        constexpr int R = CH::REM ? CH::REM : 16;
                        wgmma_rs<R, 1>(acc + CH::col(c) / 2, da[kk], chunk_desc_mnmajor(sq + CH::offset(c, WIDE_KT), R, kk), 1u);
                    }
                }
            }
            wgmma_commit();
            wgmma_wait<0>();
            reg_fence<HD / 2>(acc);
            __syncwarp();
            mbar_arrive_lane0(&qd_empty[s], lane);
            if (++s == WIDE_STAGES) s = 0, ph ^= 1;
        }
    }

    // ---------------- dV (A) or dK (B) -> its slot of dqkv ----------------
    const int col = wg == 1 ? v_col : k_col;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        if (kr[h] >= loc.doc_len) continue;
        __nv_bfloat16* row = p.dqkv + (loc.doc_start + int64_t(kr[h])) * p.row_stride + col + wc;
#pragma unroll
        for (int b = 0; b < HD / 8; ++b)
            *reinterpret_cast<uint32_t*>(row + 8 * b) = pack_bf16(acc[4 * b + 2 * h], acc[4 * b + 2 * h + 1]);
    }
}

// ================================================================================================================
// backward: dQ
// ================================================================================================================
// One CTA = 64 query rows (one half of a 128-query tile) of one head of one document: one consumer warpgroup (warpgroup 1)
// walks the 64-key tiles its queries see, in order, as attn_dq_kernel does --
//     S = Q K_j^T, dP = dO V_j^T (SS)   dS = scale * P o (Z o dP - Delta)   dQ += dS K_j (RS)
// with the SS group of key tile j + 1 issued right behind the RS group of key tile j below head_dim 256 -- and an elected lane of warpgroup 0
// streams (K_j, V_j) through the ring.  Per thread at head_dim 256: dQ 128 + S 16 + dP 16 + dS fragments 8 (see KH).  The
// warpgroups start with setmaxnreg, as in attn_dq_kernel: without an aligned instruction on the consumer's path ptxas
// treats it as divergent and serialises its wgmmas.
constexpr int WDQ_THREADS = 256;
constexpr int WDQ_CONSUMER_REGS = 256;
static_assert(WIDE_PRODUCER_REGS * 128 + WDQ_CONSUMER_REGS * 128 <= 65536, "register file exceeded");

// dS (into sc) of the KH keys from k0 on, from S, dP; MASK = test causality and the document end per element
template <bool ALIBI, bool MASK, int KH>
__device__ __forceinline__ void wide_dq_ds(float (&sc)[KH / 2], const float (&dp)[KH / 2], const WideParams& p,
                                           const TileLoc& loc, int k0, int wc, const int (&qr)[2], const float (&lse_r)[2],
                                           const float (&del_r)[2], float slope, uint32_t head_key, bool drop) {
#pragma unroll
    for (int b = 0; b < KH / 8; ++b)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int k = k0 + 8 * b + wc + e;
            const float bl = ALIBI ? attn_alibi_bias(slope, k) * ATT_LOG2E : 0.f;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int i = 4 * b + 2 * h + e;
                const bool ok = !MASK || (k <= qr[h] && qr[h] < loc.doc_len);  // causal, and a real query of the document
                float pr;
                if constexpr (ALIBI)
                    pr = ok ? fast_exp2(fmaf(sc[i], p.scale_log2, bl) - lse_r[h]) : 0.f;
                else
                    pr = ok ? fast_exp2(fmaf(sc[i], p.scale_log2, -lse_r[h])) : 0.f;
                float d = dp[i];
                if (drop) d *= attn_drop_scale(p.drop, head_key, loc.doc_start + qr[h], loc.doc_start + k);
                sc[i] = p.scale * pr * (d - del_r[h]);
            }
        }
}

template <int HD, bool ALIBI>
__global__ void __launch_bounds__(WDQ_THREADS, 1)
    attn_wide_dq_kernel(const __grid_constant__ CUtensorMap tq64, const __grid_constant__ CUtensorMap tqR,
                        const __grid_constant__ CUtensorMap to64, const __grid_constant__ CUtensorMap toR,
                        const WideParams p) {
    using CH = HeadChunks<HD>;
    constexpr int T_BYTES = CH::tile_bytes(WIDE_KT);
    // keys per MMA step: at head_dim 256, dQ 128 + S 32 + dP 32 per thread leave too few of the 255 registers, so each 64-key
    // tile runs as two 32-key steps on the same shared-memory tile, one group after the other; below 256 one step per tile,
    // with the SS group of key tile j + 1 issued behind the RS group of key tile j.  ptxas serialises the wgmmas of the
    // two-step instances (C7515, accumulator registers defined by non-wgmma instructions); DESIGN.md section 7 has the cost
    constexpr int KH = HD < 256 ? WIDE_KT : WIDE_KT / 2;
    constexpr int NKH = WIDE_KT / KH;
    constexpr bool SS_AHEAD = NKH == 1;

    int half, head;
    attn_cta_order(p.head_chunk, p.n_slots, half, head);
    half = p.n_slots - 1 - half;  // long (late) tiles first
    const TileLoc loc = locate_tile(p.cu_seqlens, p.n_docs, half >> 1);
    if (!loc.valid) return;
    const int q0 = loc.tile * ATT_TILE + (half & 1) * WIDE_KT;  // first query (doc-relative) of this CTA
    if (q0 >= loc.doc_len) return;
    const int group = head / p.q_per_group, slot = head % p.q_per_group;
    const int q_col = (group * (p.q_per_group + 2) + slot) * HD;
    const int k_col = (group * (p.q_per_group + 2) + p.q_per_group) * HD;
    const int v_col = k_col + HD;
    const int n_kt = q0 / WIDE_KT + 1;  // causal: key tiles 0 .. the diagonal one

    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_align_1024(smem_raw);
    uint8_t* sQ = smem;
    uint8_t* sO = sQ + T_BYTES;                 // dO
    uint8_t* sK = sO + T_BYTES;                 // [WIDE_STAGES]
    uint8_t* sV = sK + WIDE_STAGES * T_BYTES;   // [WIDE_STAGES]
    uint64_t* bars = reinterpret_cast<uint64_t*>(sV + WIDE_STAGES * T_BYTES);
    uint64_t* q_full = bars;                       // 1
    uint64_t* kv_full = bars + 1;                  // [WIDE_STAGES]
    uint64_t* kv_empty = bars + 1 + WIDE_STAGES;   // [WIDE_STAGES], one arrive per consumer warp

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tq64);
        tma_prefetch_desc(&to64);
        if (CH::REM > 0) {
            tma_prefetch_desc(&tqR);
            tma_prefetch_desc(&toR);
        }
        mbar_init(q_full, 1);
        for (int i = 0; i < WIDE_STAGES; ++i) {
            mbar_init(&kv_full[i], 1);
            mbar_init(&kv_empty[i], 4);  // one arrive per consumer warp
        }
        mbar_fence_init();
        mbar_expect_tx(q_full, 2 * T_BYTES);
        tma_load_chunked<HD, WIDE_KT>(sQ, &tq64, &tqR, q_full, q_col, loc.doc_start + q0);
        tma_load_chunked<HD, WIDE_KT>(sO, &to64, &toR, q_full, head * HD, loc.doc_start + q0);
    }
    __syncthreads();

    if (warp < 4) {
        // ================= producer =================
        setmaxnreg_dec<WIDE_PRODUCER_REGS>();
        if (warp == 0 && elect_one()) {
            int s = 0;
            uint32_t ph = 0;
            for (int j = 0; j < n_kt; ++j) {
                mbar_wait(&kv_empty[s], ph ^ 1, 65);
                mbar_expect_tx(&kv_full[s], 2 * T_BYTES);
                tma_load_chunked<HD, WIDE_KT>(sK + s * T_BYTES, &tq64, &tqR, &kv_full[s], k_col, loc.doc_start + j * WIDE_KT);
                tma_load_chunked<HD, WIDE_KT>(sV + s * T_BYTES, &tq64, &tqR, &kv_full[s], v_col, loc.doc_start + j * WIDE_KT);
                if (++s == WIDE_STAGES) s = 0, ph ^= 1;
            }
        }
        return;
    }

    // ================= consumer warpgroup: queries [q0, q0 + 64) =================
    setmaxnreg_inc<WDQ_CONSUMER_REGS>();
    const int n_kt_u = __shfl_sync(0xffffffffu, n_kt, 0);  // warp-uniform to ptxas: the loop branches with an SS group in flight
    const int wr = (warp & 3) * 16 + (lane >> 2);
    const int wc = 2 * (lane & 3);
    const int qr[2] = {q0 + wr, q0 + wr + 8};
    const bool drop = p.drop.threshold != 0;
    const uint32_t head_key = dropout_head_key(uint32_t(head), p.drop.key0, p.drop.key1);
    const float slope = ALIBI ? __ldg(p.alibi_slopes + head) : 0.f;
    float lse_r[2], del_r[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const bool ok = qr[h] < loc.doc_len;
        const int64_t idx = int64_t(head) * p.T + loc.doc_start + qr[h];
        lse_r[h] = ok ? __ldg(p.lse + idx) * ATT_LOG2E : 0.f;
        del_r[h] = ok ? __ldg(p.delta + idx) : 0.f;
    }
    // key tiles j >= j_diag test the predicate: the diagonal one, or all of them if the rows cross the document end
    const int j_diag = (q0 + WIDE_KT > loc.doc_len) ? 0 : q0 / WIDE_KT;
    const uint32_t sq = smem_u32(sQ), so = smem_u32(sO);
    float dq[HD / 2];
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) dq[i] = 0.f;
    float sc[KH / 2], dp[KH / 2];

    // S, dP of keys [kh * KH, kh * KH + KH) of the key tile in ring stage s (one commit group)
    auto issue_ss = [&](int s, int kh) {
        uint32_t sk = smem_u32(sK + s * T_BYTES), sv = smem_u32(sV + s * T_BYTES);
        opaque(sk), opaque(sv);
        wgmma_fence();
#pragma unroll
        for (int c = 0; c < CH::NCHUNK; ++c) {
            const int w = CH::width(c);
            const uint32_t krow = CH::offset(c, WIDE_KT) + kh * KH * 2 * w;
#pragma unroll
            for (int k = 0; k < w / 16; ++k) {
                wgmma_ss<KH, 0, 0>(sc, chunk_desc_kmajor(sq + CH::offset(c, WIDE_KT), w, k), chunk_desc_kmajor(sk + krow, w, k),
                                   (c != 0 || k != 0) ? 1u : 0u);
                wgmma_ss<KH, 0, 0>(dp, chunk_desc_kmajor(so + CH::offset(c, WIDE_KT), w, k), chunk_desc_kmajor(sv + krow, w, k),
                                   (c != 0 || k != 0) ? 1u : 0u);
            }
        }
        wgmma_commit();
    };

    mbar_spin(q_full, 0);
    int s = 0;
    uint32_t ph = 0;
    mbar_spin(&kv_full[0], 0);
    issue_ss(0, 0);
    for (int j = 0; j < n_kt_u; ++j) {
        const int s1 = s + 1 == WIDE_STAGES ? 0 : s + 1;
        const uint32_t ph1 = s1 == 0 ? ph ^ 1 : ph;
        const bool more = j + 1 < n_kt_u;
#pragma unroll
        for (int kh = 0; kh < NKH; ++kh) {
            wgmma_wait<0>();
            reg_fence<KH / 2>(sc);
            reg_fence<KH / 2>(dp);
            const int kb = j * WIDE_KT + kh * KH;
            if (j >= j_diag)
                wide_dq_ds<ALIBI, true, KH>(sc, dp, p, loc, kb, wc, qr, lse_r, del_r, slope, head_key, drop);
            else
                wide_dq_ds<ALIBI, false, KH>(sc, dp, p, loc, kb, wc, qr, lse_r, del_r, slope, head_key, drop);
            uint32_t da[KH / 16][4];
#pragma unroll
            for (int kk = 0; kk < KH / 16; ++kk) acc_to_a_frag(sc, kk, da[kk]);

            if (kh + 1 == NKH && more) mbar_spin(&kv_full[s1], ph1);
            uint32_t sk = smem_u32(sK + s * T_BYTES);
            opaque(sk);
            wgmma_fence();
#pragma unroll
            for (int c = 0; c < CH::NCHUNK; ++c) {
#pragma unroll
                for (int kk = 0; kk < KH / 16; ++kk) {
                    const int k16 = kh * (KH / 16) + kk;  // 16-key group of the tile
                    if (CH::width(c) == 64) {
                        wgmma_rs<64, 1>(dq + CH::col(c) / 2, da[kk], chunk_desc_mnmajor(sk + CH::offset(c, WIDE_KT), 64, k16), 1u);
                    } else {
                        constexpr int R = CH::REM ? CH::REM : 16;
                        wgmma_rs<R, 1>(dq + CH::col(c) / 2, da[kk], chunk_desc_mnmajor(sk + CH::offset(c, WIDE_KT), R, k16), 1u);
                    }
                }
            }
            wgmma_commit();

            if (SS_AHEAD && more) {
                issue_ss(s1, 0);
                wgmma_wait<1>();  // the RS group of key tile j is done; the SS group of key tile j + 1 runs on
            } else {
                wgmma_wait<0>();
            }
            reg_fence<HD / 2>(dq);
            if (!SS_AHEAD) {
                if (kh + 1 < NKH)
                    issue_ss(s, kh + 1);
                else if (more)
                    issue_ss(s1, 0);
            }
        }
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
int launch_wide_bwd(const void* dout, const void* qkv, int64_t row_stride, WideParams p, int head_chunk_kv,
                    int head_chunk_q, cudaStream_t st) {
    using CH = HeadChunks<HD>;
    CUtensorMap tq64, tqR, to64, toR;
    int rc = attn_make_maps<HD>(qkv, row_stride, p.T, &tq64, &tqR);
    if (rc) return rc;
    rc = attn_make_maps<HD>(dout, int64_t(p.n_heads) * HD, p.T, &to64, &toR);
    if (rc) return rc;
    constexpr int T_BYTES = CH::tile_bytes(WIDE_KT);
    constexpr int bwd_smem = 1024 + 2 * T_BYTES + 2 * WIDE_STAGES * T_BYTES + WIDE_KT * WIDE_KT * 4 +
                             WIDE_STAGES * 2 * WIDE_KT * 4 + 128;
    static_assert(bwd_smem <= 232448, "wide attention dK/dV shared memory budget exceeded");
    constexpr int dq_smem = 1024 + 2 * T_BYTES + 2 * WIDE_STAGES * T_BYTES + 128;
    static_assert(dq_smem <= 232448, "wide attention dQ shared memory budget exceeded");
    auto kb = attn_wide_bwd_kernel<HD, ALIBI>;
    auto kq = attn_wide_dq_kernel<HD, ALIBI>;
    static bool attr_set = false;
    if (!attr_set) {
        DOLO_CUDA_OK(cudaFuncSetAttribute(kb, cudaFuncAttributeMaxDynamicSharedMemorySize, bwd_smem));
        DOLO_CUDA_OK(cudaFuncSetAttribute(kq, cudaFuncAttributeMaxDynamicSharedMemorySize, dq_smem));
        attr_set = true;
    }
    DOLO_REQUIRE(int64_t(p.n_slots) * p.n_heads < (1ll << 31), "attn_bwd: grid too large");
    p.head_chunk = head_chunk_kv;
    kb<<<dim3(unsigned(p.n_slots * p.n_groups)), WBWD_THREADS, bwd_smem, st>>>(tq64, tqR, to64, toR, p);
    DOLO_LAUNCH_OK("attn_varlen_bwd");
    p.head_chunk = head_chunk_q;
    kq<<<dim3(unsigned(p.n_slots * p.n_heads)), WDQ_THREADS, dq_smem, st>>>(tq64, tqR, to64, toR, p);
    DOLO_LAUNCH_OK("attn_varlen_bwd_dq");
    return DOLO_OK;
}

// ================================================================================================================
// decode
// ================================================================================================================
// attn_decode_kernel with 256 threads: 256 keys per chunk in phase A, one output column per thread in phase B.
constexpr int WDEC_THREADS = 256;

template <int HD, bool ALIBI>
__global__ void __launch_bounds__(WDEC_THREADS)
    attn_wide_decode_kernel(const __nv_bfloat16* __restrict__ qkv, int64_t row_stride,
                            const __nv_bfloat16* __restrict__ k_cache, const __nv_bfloat16* __restrict__ v_cache,
                            const int32_t* __restrict__ lens, __nv_bfloat16* __restrict__ out, int64_t L_max, int n_groups,
                            int q_per_group, float scale_log2, const float* __restrict__ alibi_slopes) {
    static_assert(HD % 8 == 0 && HD <= WDEC_THREADS, "one thread per output column");
    __shared__ __align__(16) float sq[HD];
    __shared__ float sp[WDEC_THREADS];
    __shared__ float red[WDEC_THREADS / 32];
    __shared__ float s_bcast[2];
    const int b = blockIdx.x, head = blockIdx.y;
    const int group = head / q_per_group, slot = head % q_per_group;
    const int n_heads = n_groups * q_per_group;
    const int len = lens[b];
    const int t = threadIdx.x, lane = t & 31, wid = t >> 5;
    const __nv_bfloat16* q = qkv + int64_t(b) * row_stride + int64_t(group * (q_per_group + 2) + slot) * HD;
    if (t < HD) sq[t] = __bfloat162float(q[t]);
    __syncthreads();
    const int64_t kv_stride = int64_t(n_groups) * HD;  // elements between consecutive positions
    const __nv_bfloat16* kb = k_cache + (int64_t(b) * L_max) * kv_stride + int64_t(group) * HD;
    const __nv_bfloat16* vb = v_cache + (int64_t(b) * L_max) * kv_stride + int64_t(group) * HD;
    float m_run = -INFINITY, l_run = 0.f, acc = 0.f;
    const float slope = ALIBI ? __ldg(alibi_slopes + head) : 0.f;
    for (int base = 0; base < len; base += WDEC_THREADS) {
        // ---- phase A: one key per thread ----
        const int key = base + t;
        float s = -INFINITY;
        if (key < len) {
            const uint4* kr = reinterpret_cast<const uint4*>(kb + int64_t(key) * kv_stride);
            float dot = 0.f;
#pragma unroll
            for (int v = 0; v < HD / 8; ++v) {
                const uint4 kk = __ldg(kr + v);
                const float4 qa = *reinterpret_cast<const float4*>(sq + v * 8);
                const float4 qb = *reinterpret_cast<const float4*>(sq + v * 8 + 4);
                dot += bf16_lo(kk.x) * qa.x + bf16_hi(kk.x) * qa.y + bf16_lo(kk.y) * qa.z + bf16_hi(kk.y) * qa.w;
                dot += bf16_lo(kk.z) * qb.x + bf16_hi(kk.z) * qb.y + bf16_lo(kk.w) * qb.z + bf16_hi(kk.w) * qb.w;
            }
            if constexpr (ALIBI)
                s = fmaf(dot, scale_log2, attn_alibi_bias(slope, key) * ATT_LOG2E);
            else
                s = dot * scale_log2;  // log2 units
        }
        float cm = warp_max(s);
        if (lane == 0) red[wid] = cm;
        __syncthreads();
        if (t == 0) {
            float mm = red[0];
#pragma unroll
            for (int i = 1; i < WDEC_THREADS / 32; ++i) mm = fmaxf(mm, red[i]);
            s_bcast[0] = fmaxf(m_run, mm);
        }
        __syncthreads();
        const float m_new = s_bcast[0];
        const float alpha = (m_run == -INFINITY) ? 0.f : fast_exp2(m_run - m_new);
        const float p = (key < len) ? fast_exp2(s - m_new) : 0.f;
        sp[t] = p;
        float cs = warp_sum(p);
        __syncthreads();  // red[] / s_bcast[0] consumed by everyone, sp[] complete after the next barrier
        if (lane == 0) red[wid] = cs;
        __syncthreads();
        float csum = 0.f;
#pragma unroll
        for (int i = 0; i < WDEC_THREADS / 32; ++i) csum += red[i];
        l_run = l_run * alpha + csum;
        m_run = m_new;
        // ---- phase B: one output column per thread ----
        if (t < HD) {
            const int n = min(WDEC_THREADS, len - base);
            float a = acc * alpha;
            const __nv_bfloat16* vcol = vb + int64_t(base) * kv_stride + t;
#pragma unroll 4
            for (int k = 0; k < n; ++k) a = fmaf(sp[k], __bfloat162float(vcol[int64_t(k) * kv_stride]), a);
            acc = a;
        }
        __syncthreads();  // sp[] / red[] are rewritten by the next chunk
    }
    if (t < HD) out[int64_t(b) * (int64_t(n_heads) * HD) + int64_t(head) * HD + t] = __float2bfloat16_rn(l_run > 0.f ? acc / l_run : 0.f);
}

template <int HD>
int launch_wide_decode(const void* qkv, int64_t row_stride, const void* k_cache, const void* v_cache, const int32_t* lens,
                       void* out, int B, int64_t L_max, int n_groups, int q_per_group, float scale, const float* alibi_slopes,
                       cudaStream_t st) {
    dim3 grid((unsigned)B, (unsigned)(n_groups * q_per_group));
    auto kern = alibi_slopes != nullptr ? attn_wide_decode_kernel<HD, true> : attn_wide_decode_kernel<HD, false>;
    kern<<<grid, WDEC_THREADS, 0, st>>>(static_cast<const __nv_bfloat16*>(qkv), row_stride,
                                        static_cast<const __nv_bfloat16*>(k_cache), static_cast<const __nv_bfloat16*>(v_cache),
                                        lens, static_cast<__nv_bfloat16*>(out), L_max, n_groups, q_per_group,
                                        scale * 1.4426950408889634f, alibi_slopes);
    DOLO_LAUNCH_OK("attn_decode");
    return DOLO_OK;
}

WideParams wide_params(const int32_t* cu_seqlens, int n_docs, int64_t T, int n_groups, int q_per_group, float softmax_scale,
                       float dropout_p, uint32_t key0, uint32_t key1, const float* alibi_slopes) {
    WideParams p{};
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
    p.alibi_slopes = alibi_slopes;
    return p;
}

}  // namespace

int dolo_attn_wide_fwd(const void* qkv, int64_t row_stride, void* out, float* lse, const int32_t* cu_seqlens, int n_docs,
                       int64_t T, int n_groups, int q_per_group, int head_dim, float softmax_scale, float dropout_p,
                       uint32_t key0, uint32_t key1, const float* alibi_slopes, cudaStream_t st) {
    WideParams p = wide_params(cu_seqlens, n_docs, T, n_groups, q_per_group, softmax_scale, dropout_p, key0, key1,
                               alibi_slopes);
    p.out = static_cast<__nv_bfloat16*>(out);
    p.lse_out = lse;
    p.n_slots = int((T + ATT_TILE - 1) / ATT_TILE + n_docs);
    p.head_chunk = attn_head_chunk(dolo_option_attn_head_fastest(), p.n_heads, q_per_group);
    // all heads in one chunk when the K / V of the whole batch stay in L2 anyway (as attn_fwd)
    if (p.head_chunk > 0 && T * int64_t(n_groups) * head_dim * 4 <= (24ll << 20)) p.head_chunk = p.n_heads;
    const bool ab = alibi_slopes != nullptr;
    switch (head_dim) {
        case 160: return ab ? launch_wide_fwd<160, true>(qkv, row_stride, p, st) : launch_wide_fwd<160, false>(qkv, row_stride, p, st);
        case 192: return ab ? launch_wide_fwd<192, true>(qkv, row_stride, p, st) : launch_wide_fwd<192, false>(qkv, row_stride, p, st);
        case 256: return ab ? launch_wide_fwd<256, true>(qkv, row_stride, p, st) : launch_wide_fwd<256, false>(qkv, row_stride, p, st);
        default: return dolo_set_error("attn_fwd: no wide kernel for head_dim %d", head_dim);
    }
}

int dolo_attn_wide_bwd(const void* dout, const void* qkv, int64_t row_stride, const float* lse, const float* delta,
                       void* dqkv, const int32_t* cu_seqlens, int n_docs, int64_t T, int n_groups, int q_per_group,
                       int head_dim, float softmax_scale, float dropout_p, uint32_t key0, uint32_t key1,
                       const float* alibi_slopes, cudaStream_t st) {
    WideParams p = wide_params(cu_seqlens, n_docs, T, n_groups, q_per_group, softmax_scale, dropout_p, key0, key1,
                               alibi_slopes);
    p.lse = lse;
    p.delta = delta;
    p.dqkv = static_cast<__nv_bfloat16*>(dqkv);
    p.row_stride = row_stride;
    p.n_slots = int(2 * ((T + ATT_TILE - 1) / ATT_TILE + n_docs));
    const int chunk_kv = attn_head_chunk(dolo_option_attn_head_fastest(), n_groups, 1);
    const int chunk_q = attn_head_chunk(dolo_option_attn_head_fastest(), p.n_heads, q_per_group);
    const bool ab = alibi_slopes != nullptr;
    switch (head_dim) {
        case 160: return ab ? launch_wide_bwd<160, true>(dout, qkv, row_stride, p, chunk_kv, chunk_q, st)
                            : launch_wide_bwd<160, false>(dout, qkv, row_stride, p, chunk_kv, chunk_q, st);
        case 192: return ab ? launch_wide_bwd<192, true>(dout, qkv, row_stride, p, chunk_kv, chunk_q, st)
                            : launch_wide_bwd<192, false>(dout, qkv, row_stride, p, chunk_kv, chunk_q, st);
        case 256: return ab ? launch_wide_bwd<256, true>(dout, qkv, row_stride, p, chunk_kv, chunk_q, st)
                            : launch_wide_bwd<256, false>(dout, qkv, row_stride, p, chunk_kv, chunk_q, st);
        default: return dolo_set_error("attn_bwd: no wide kernel for head_dim %d", head_dim);
    }
}

int dolo_attn_wide_decode(const void* qkv, int64_t row_stride, const void* k_cache, const void* v_cache,
                          const int32_t* lens, void* out, int batch, int64_t L_max, int n_groups, int q_per_group,
                          int head_dim, float softmax_scale, const float* alibi_slopes, cudaStream_t st) {
    switch (head_dim) {
        case 160: return launch_wide_decode<160>(qkv, row_stride, k_cache, v_cache, lens, out, batch, L_max, n_groups, q_per_group, softmax_scale, alibi_slopes, st);
        case 192: return launch_wide_decode<192>(qkv, row_stride, k_cache, v_cache, lens, out, batch, L_max, n_groups, q_per_group, softmax_scale, alibi_slopes, st);
        case 256: return launch_wide_decode<256>(qkv, row_stride, k_cache, v_cache, lens, out, batch, L_max, n_groups, q_per_group, softmax_scale, alibi_slopes, st);
        default: return dolo_set_error("attn_decode: no wide kernel for head_dim %d", head_dim);
    }
}
