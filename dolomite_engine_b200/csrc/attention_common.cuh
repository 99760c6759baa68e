// Shared pieces of the packed var-len causal attention kernels (forward and backward).
//
// qkv slot layout (reference: attention/padding_free.py:79-116): each token row holds `n_groups` groups of
// (q_per_group + 2) head slots of head_dim bf16: [q_0 .. q_{g-1}, k, v].  mha: n_groups = n_head, g = 1;
// gqa: n_groups = n_kv, g = n_head / n_kv; mqa: n_groups = 1, g = n_head.
//
// A [rows x head_dim] tile of Q, K, V or dO is staged in shared memory as "chunks" along head_dim so that each chunk is
// one TMA box (64 rows per box) with a hardware swizzle that wgmma understands:  64-wide chunks (128 B rows, SWIZZLE_128B)
// followed by one remainder chunk of 32 (SWIZZLE_64B) or 16 (SWIZZLE_32B) columns.  head_dim 80 = 64 + 16, 128 = 64 + 64.
// The same bytes serve as a K-major operand (rows = MMA M/N, head_dim = contraction) and as an MN-major operand
// (head_dim = MMA N, rows = contraction), only the descriptor differs.
#pragma once
#include "common.cuh"
#include "wgmma.cuh"
#include "../../include/dolomite_b200.h"

namespace dolo {

constexpr int ATT_TILE = 128;  // query rows (forward) / key rows (backward) per CTA tile

template <int HD>
struct HeadChunks {
    static_assert(HD % 16 == 0 && HD >= 16 && HD <= 256, "head_dim must be a multiple of 16 in [16, 256]");
    static constexpr int NC64 = HD / 64;
    static constexpr int REM = HD % 64;
    static_assert(REM == 0 || REM == 16 || REM == 32, "head_dim % 64 must be 0, 16 or 32");
    static constexpr int NCHUNK = NC64 + (REM ? 1 : 0);
    __host__ __device__ static constexpr int width(int c) { return c < NC64 ? 64 : REM; }
    __host__ __device__ static constexpr int col(int c) { return c * 64; }  // first head_dim column of chunk
    // byte offset of chunk c inside a tile of `rows` rows (a full chunk is rows x 128 B)
    __host__ __device__ static constexpr int offset(int c, int rows) { return c * rows * 128; }
    __host__ __device__ static constexpr int tile_bytes(int rows) { return rows * HD * 2; }
};

// wgmma layout_type field for a chunk of `w` bf16 columns
__host__ __device__ constexpr uint32_t chunk_layout_type(int w) { return w == 64 ? 1u : (w == 32 ? 2u : 3u); }

// K-major view of a chunk (rows = M or N of the MMA, chunk columns = contraction), k16 = which 16-wide K step
__device__ __forceinline__ uint64_t chunk_desc_kmajor(uint32_t chunk_saddr, int w, int k16) {
    return gmma_desc(chunk_saddr + k16 * 32, 16, 16 * w, chunk_layout_type(w));
}
// MN-major view (chunk columns = N of the MMA, rows = contraction), k16 = which group of 16 rows
__device__ __forceinline__ uint64_t chunk_desc_mnmajor(uint32_t chunk_saddr, int w, int k16) {
    return gmma_desc(chunk_saddr + k16 * 32 * w, 16 * w, 16 * w, chunk_layout_type(w));
}

// TMA of a [ROWS x HD] tile (columns col0.., rows row0..) into the chunked layout, in boxes of 64 rows; m64 / mR are the
// maps of the 64-wide and of the remainder chunks.  Rows past the tensor are zero-filled by the TMA unit.
template <int HD, int ROWS>
__device__ __forceinline__ void tma_load_chunked(uint8_t* dst, const CUtensorMap* m64, const CUtensorMap* mR, uint64_t* bar,
                                                 int col0, int row0) {
    using CH = HeadChunks<HD>;
#pragma unroll
    for (int c = 0; c < CH::NCHUNK; ++c)
#pragma unroll
        for (int h = 0; h < ROWS / 64; ++h)
            tma_load_2d(dst + CH::offset(c, ROWS) + h * 64 * 2 * CH::width(c), c < CH::NC64 ? m64 : mR, bar,
                        col0 + CH::col(c), row0 + h * 64);
}

// the two tensor maps (64-wide chunks / remainder chunk, 64-row boxes) of a bf16 [rows, ld] matrix
template <int HD>
int attn_make_maps(const void* base, int64_t ld, int64_t rows, CUtensorMap* m64, CUtensorMap* mR) {
    using CH = HeadChunks<HD>;
    uint64_t dims[2] = {uint64_t(ld), uint64_t(rows)};
    uint64_t strides[2] = {2, uint64_t(ld) * 2};
    uint32_t box[2] = {64, 64};
    int rc;
    if (CH::NC64 > 0) {
        rc = dolo_make_tmap(m64, base, 2, 2, dims, strides, box, DOLO_SW_128);
        if (rc) return rc;
    }
    if (CH::REM > 0) {
        box[0] = CH::REM;
        rc = dolo_make_tmap(mR, base, 2, 2, dims, strides, box, CH::REM == 32 ? DOLO_SW_64 : DOLO_SW_32);
        if (rc) return rc;
    }
    if (CH::NC64 == 0) *m64 = *mR;
    if (CH::REM == 0) *mR = *m64;
    return DOLO_OK;
}

// Attention-probability dropout (attention/base.py:252 `attn_dropout`; flash_attn_varlen_func(dropout_p=...) at
// attention/padding_free.py:49-59): P_ij is kept with probability 1 - p and scaled by 1 / (1 - p) AFTER the softmax
// normaliser was taken over the undropped row.  The mask is a hash of (global query token, global key token, head) and the
// keys of the call site, so the backward kernels regenerate it.  threshold == 0 <=> no dropout.
struct AttnDropout {
    uint32_t threshold;
    float keep_scale;
    uint32_t key0, key1;
};
__device__ __forceinline__ float attn_drop_scale(const AttnDropout& d, uint32_t head_key, int q_tok, int k_tok) {
    return dropout_hash_qk(uint32_t(q_tok), uint32_t(k_tok), head_key) >= d.threshold ? d.keep_scale : 0.f;
}

// ALiBi (modeling_utils/position_embedding/alibi.py:14-30, gpt_dolomite/base.py:261-287): the logit of (query, key) of
// head h gets bias = slope_h * kpos, where kpos is the key's index inside its document (the packed form of
// `cumsum(attention_mask) - 1`) or inside the KV cache.  The reference casts the bias to the hidden-state dtype, so it is
// bf16(fp32(slope) * kpos); the slopes are the reference's fp32 values, computed on the host.
__device__ __forceinline__ float attn_alibi_bias(float slope, int kpos) {
    return __bfloat162float(__float2bfloat16_rn(slope * float(kpos)));
}
constexpr float ATT_LOG2E = 1.4426950408889634f;
constexpr float ATT_LN2 = 0.6931471805599453f;

// CTA order of the attention grids (1-D grid of n_tile_slots x n_heads CTAs, dispatched in index order).  Heads are taken
// in CHUNKS of `chunk`; inside a chunk the heads are the fastest index and the tile the slower one, and the callers walk the
// tiles of a document longest first.  The last wave of a chunk then holds short tiles only and the next chunk's long tiles
// start while they drain; with tiles fastest (chunk == 0) the LONG tiles of the last heads start in the last wave, and with
// few waves that tail is large.  With every head in one chunk, though, only a few CTAs of a head run at a time and each
// re-reads the head's K / V (forward) or Q / dO (backward) stream from DRAM; chunks of 8 heads keep the CTAs of a head on
// one stream in L2.
__device__ __forceinline__ void attn_cta_order(int chunk, int n_tile_slots, int& tile, int& head) {
    const int id = int(blockIdx.x);
    if (chunk <= 0) {  // tiles fastest
        tile = id % n_tile_slots;
        head = id / n_tile_slots;
        return;
    }
    const int per = n_tile_slots * chunk;
    const int c = id / per, r = id - c * per;
    tile = r / chunk;
    head = c * chunk + (r - tile * chunk);
}
// heads per chunk for `n` heads (kv groups in the backward): the option value rounded to a divisor of n that keeps the q
// heads of a kv group together (forward, `align` = q_per_group); 0 = tiles fastest
inline int attn_head_chunk(int option, int n, int align) {
    if (option <= 0 || n <= 0) return 0;
    if (align < 1 || n % align != 0) align = 1;
    int best = 0;
    for (int c = align; c <= n; c += align)
        if (n % c == 0 && c <= (option > align ? option : align)) best = c;
    return best > 0 ? best : n;
}

// Hides a shared-memory base address from the compiler's loop-invariant code motion, so that the wgmma descriptors built
// from it are recomputed next to each MMA instead of being hoisted out of the step loop and held in registers.
__device__ __forceinline__ void opaque(uint32_t& x) { asm volatile("" : "+r"(x)); }
// Wait without the watchdog of mbar_wait, for waits with an MMA group in flight: ptxas serialises every wgmma of a kernel
// that has a trap path (or any other divergent branch) while a group is in flight.
__device__ __forceinline__ void mbar_spin(uint64_t* bar, uint32_t parity) {
    asm volatile("{\n\t.reg .pred P1;\n\tWAIT_%=:\n\tmbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t@!P1 bra WAIT_%=;\n\t}"
                 ::"r"(smem_u32(bar)), "r"(parity)
                 : "memory");
}
// Arrive of lane 0 only, as a predicated instruction rather than a branch, for the same reason.
__device__ __forceinline__ void mbar_arrive_lane0(uint64_t* bar, int lane) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.eq.s32 p, %1, 0;\n\t@p mbarrier.arrive.shared::cta.b64 _, [%0];\n\t}" ::"r"(smem_u32(bar)),
                 "r"(lane)
                 : "memory");
}

// Locate the (document, q-tile) of a linear tile index by scanning cu_seqlens (B is small: a few docs per row).
struct TileLoc {
    int doc_start;  // first token of the document
    int doc_len;
    int tile;       // 128-row tile index inside the document
    bool valid;
};
__device__ __forceinline__ TileLoc locate_tile(const int32_t* __restrict__ cu, int n_docs, int ti) {
    TileLoc r{0, 0, 0, false};
    int acc = 0;
    for (int d = 0; d < n_docs; ++d) {
        const int s = cu[d], e = cu[d + 1];
        const int nt = (e - s + ATT_TILE - 1) / ATT_TILE;
        if (ti < acc + nt) {
            r.doc_start = s;
            r.doc_len = e - s;
            r.tile = ti - acc;
            r.valid = true;
            return r;
        }
        acc += nt;
    }
    return r;
}

}  // namespace dolo

// Wide heads (head_dim 160, 192, 256; attention_wide.cu): the launches behind the head_dim switches of the attention entry
// points, called after those have checked their arguments.  Same arguments and semantics as the narrow kernels'.
int dolo_attn_wide_fwd(const void* qkv, int64_t row_stride, void* out, float* lse, const int32_t* cu_seqlens, int n_docs,
                       int64_t T, int n_groups, int q_per_group, int head_dim, float softmax_scale, float dropout_p,
                       uint32_t key0, uint32_t key1, const float* alibi_slopes, cudaStream_t st);
// dK / dV and dQ, given Delta (attn_delta_kernel) in `delta` [n_heads, T]
int dolo_attn_wide_bwd(const void* dout, const void* qkv, int64_t row_stride, const float* lse, const float* delta,
                       void* dqkv, const int32_t* cu_seqlens, int n_docs, int64_t T, int n_groups, int q_per_group,
                       int head_dim, float softmax_scale, float dropout_p, uint32_t key0, uint32_t key1,
                       const float* alibi_slopes, cudaStream_t st);
int dolo_attn_wide_decode(const void* qkv, int64_t row_stride, const void* k_cache, const void* v_cache,
                          const int32_t* lens, void* out, int batch, int64_t L_max, int n_groups, int q_per_group,
                          int head_dim, float softmax_scale, const float* alibi_slopes, cudaStream_t st);
