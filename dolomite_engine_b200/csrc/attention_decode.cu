// Single-query attention over a KV cache (autoregressive decoding; reference: attention/sdpa.py:11-83 and
// attention/flash.py:16-140 with `past_key_values`, one new token per sequence).
//
// HBM-bound by construction: every step reads the whole cache of a sequence once (2 * L * n_kv * head_dim * 2 bytes per layer)
// and there is one query row per head, so the tensor cores have nothing to do.  One CTA = one (sequence, query head):
//   phase A  thread t scores key (chunk + t): s = scale * <q, K[key]> with q broadcast from shared memory (fp32), 16-byte
//            loads of the key row;  block-wide running maximum / sum (online softmax over chunks of 128 keys);
//   phase B  thread d (< head_dim) owns output column d: acc[d] = acc[d] * alpha + sum_keys p[key] * V[key][d]  -- the V row of a
//            key is read by head_dim consecutive threads, i.e. fully coalesced.
// Cache layout: k_cache / v_cache [B, L_max, n_groups * head_dim] bf16 (position-major per sequence); `lens[b]` = number of
// valid positions INCLUDING the token being decoded.  The query comes straight out of the packed c_attn output (slot layout of
// attention/padding_free.py:79-116), one row per sequence.
// ALIBI: the score of a key gets the bias of its cache position (attn_alibi_bias, attention_common.cuh): the cache holds the
// real tokens of a sequence from position 0 (hf_models/generation.py:56-79), so the position is the reference's
// `cumsum(attention_mask) - 1`.
#include "attention_common.cuh"
#include "../../include/dolomite_b200.h"

using namespace dolo;

namespace {

constexpr int DEC_THREADS = 128;

template <int HD, bool ALIBI>
__global__ void __launch_bounds__(DEC_THREADS)
    attn_decode_kernel(const __nv_bfloat16* __restrict__ qkv, int64_t row_stride, const __nv_bfloat16* __restrict__ k_cache,
                       const __nv_bfloat16* __restrict__ v_cache, const int32_t* __restrict__ lens,
                       __nv_bfloat16* __restrict__ out, int64_t L_max, int n_groups, int q_per_group, float scale_log2,
                       const float* __restrict__ alibi_slopes) {
    static_assert(HD % 8 == 0 && HD <= DEC_THREADS, "one thread per output column");
    __shared__ __align__(16) float sq[HD];
    __shared__ float sp[DEC_THREADS];
    __shared__ float red[DEC_THREADS / 32];
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
    for (int base = 0; base < len; base += DEC_THREADS) {
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
            for (int i = 1; i < DEC_THREADS / 32; ++i) mm = fmaxf(mm, red[i]);
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
        for (int i = 0; i < DEC_THREADS / 32; ++i) csum += red[i];
        l_run = l_run * alpha + csum;
        m_run = m_new;
        // ---- phase B: one output column per thread ----
        if (t < HD) {
            const int n = min(DEC_THREADS, len - base);
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

template <int HD, bool ALIBI>
int launch_decode(const void* qkv, int64_t row_stride, const void* k_cache, const void* v_cache, const int32_t* lens, void* out,
                  int B, int64_t L_max, int n_groups, int q_per_group, float scale, const float* alibi_slopes, cudaStream_t st) {
    dim3 grid((unsigned)B, (unsigned)(n_groups * q_per_group));
    attn_decode_kernel<HD, ALIBI><<<grid, DEC_THREADS, 0, st>>>(
        static_cast<const __nv_bfloat16*>(qkv), row_stride, static_cast<const __nv_bfloat16*>(k_cache),
        static_cast<const __nv_bfloat16*>(v_cache), lens, static_cast<__nv_bfloat16*>(out), L_max, n_groups, q_per_group,
        scale * 1.4426950408889634f, alibi_slopes);
    DOLO_LAUNCH_OK("attn_decode");
    return DOLO_OK;
}

}  // namespace

namespace {

template <int HD>
int launch_decode_any(const void* qkv, int64_t row_stride, const void* k_cache, const void* v_cache, const int32_t* lens,
                      void* out, int B, int64_t L_max, int n_groups, int q_per_group, float scale, const float* alibi_slopes,
                      cudaStream_t st) {
    if (alibi_slopes != nullptr)
        return launch_decode<HD, true>(qkv, row_stride, k_cache, v_cache, lens, out, B, L_max, n_groups, q_per_group, scale,
                                       alibi_slopes, st);
    return launch_decode<HD, false>(qkv, row_stride, k_cache, v_cache, lens, out, B, L_max, n_groups, q_per_group, scale,
                                    nullptr, st);
}

// alibi_slopes == nullptr: the plain kernel
int attn_decode(const void* qkv, int64_t row_stride, const void* k_cache, const void* v_cache, const int32_t* lens, void* out,
                int batch, int64_t L_max, int n_groups, int q_per_group, int head_dim, float softmax_scale,
                const float* alibi_slopes, void* stream) {
    DOLO_REQUIRE(batch >= 0 && L_max > 0, "attn_decode: bad sizes");
    if (batch == 0) return DOLO_OK;
    DOLO_REQUIRE(n_groups > 0 && q_per_group > 0, "attn_decode: bad head grouping");
    DOLO_REQUIRE(row_stride % 8 == 0 && (reinterpret_cast<uintptr_t>(qkv) & 15) == 0 &&
                     (reinterpret_cast<uintptr_t>(k_cache) & 15) == 0 && (reinterpret_cast<uintptr_t>(v_cache) & 15) == 0,
                 "attn_decode: alignment");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    switch (head_dim) {
        case 16: return launch_decode_any<16>(qkv, row_stride, k_cache, v_cache, lens, out, batch, L_max, n_groups, q_per_group, softmax_scale, alibi_slopes, st);
        case 32: return launch_decode_any<32>(qkv, row_stride, k_cache, v_cache, lens, out, batch, L_max, n_groups, q_per_group, softmax_scale, alibi_slopes, st);
        case 64: return launch_decode_any<64>(qkv, row_stride, k_cache, v_cache, lens, out, batch, L_max, n_groups, q_per_group, softmax_scale, alibi_slopes, st);
        case 80: return launch_decode_any<80>(qkv, row_stride, k_cache, v_cache, lens, out, batch, L_max, n_groups, q_per_group, softmax_scale, alibi_slopes, st);
        case 96: return launch_decode_any<96>(qkv, row_stride, k_cache, v_cache, lens, out, batch, L_max, n_groups, q_per_group, softmax_scale, alibi_slopes, st);
        case 128: return launch_decode_any<128>(qkv, row_stride, k_cache, v_cache, lens, out, batch, L_max, n_groups, q_per_group, softmax_scale, alibi_slopes, st);
        case 160: case 192: case 256:
            return dolo_attn_wide_decode(qkv, row_stride, k_cache, v_cache, lens, out, batch, L_max, n_groups, q_per_group,
                                         head_dim, softmax_scale, alibi_slopes, st);
        default: return dolo_set_error("attn_decode: unsupported head_dim %d (supported: 16,32,64,80,96,128,160,192,256)", head_dim);
    }
}

}  // namespace

extern "C" int dolomite_b200_attn_decode(const void* qkv, int64_t row_stride, const void* k_cache, const void* v_cache,
                                         const int32_t* lens, void* out, int batch, int64_t L_max, int n_groups,
                                         int q_per_group, int head_dim, float softmax_scale, void* stream) {
    return attn_decode(qkv, row_stride, k_cache, v_cache, lens, out, batch, L_max, n_groups, q_per_group, head_dim,
                       softmax_scale, nullptr, stream);
}

extern "C" int dolomite_b200_attn_decode_alibi(const void* qkv, int64_t row_stride, const void* k_cache, const void* v_cache,
                                               const int32_t* lens, void* out, int batch, int64_t L_max, int n_groups,
                                               int q_per_group, int head_dim, float softmax_scale,
                                               const float* alibi_slopes, void* stream) {
    DOLO_REQUIRE(alibi_slopes != nullptr, "attn_decode_alibi: alibi_slopes is null");
    return attn_decode(qkv, row_stride, k_cache, v_cache, lens, out, batch, L_max, n_groups, q_per_group, head_dim,
                       softmax_scale, alibi_slopes, stream);
}
