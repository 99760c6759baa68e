// bf16 and fp8 GEMM for sm_90a (H100):  TMA (cp.async.bulk.tensor) -> 128B-swizzled smem ring -> wgmma (m64n128 or
// m64n256 per consumer warpgroup, fp32 accumulators in registers) -> epilogue (scale / alpha / bias / beta*C, bf16 |
// fp32) through double-buffered shared-memory slabs -> asynchronous TMA stores.
//
// One kernel body serves both operand types; an operand policy (Bf16Ops, Fp8Ops) names what differs.  Persistent,
// warp-specialised: warpgroup 0 = producer (one elected thread issues the TMA loads; the whole first warp for
// gather-on-load), warpgroups 1 and 2 = consumers, each owning 64 rows of the output tile.  The tile is 128 x 128 (six
// 32 KB stages) or, for dense bf16 launches, 128 x 256 (four 48 KB stages; setmaxnreg moves registers from the producer
// to the consumers, which hold 128 accumulators each).  choose_tile_n picks the width per launch from the tile counts.
// bf16 operands may be K-major (row-major [rows, K]) or MN-major (stored [K, rows]); the latter is what dgrad / wgrad
// need, so no transposes are ever materialised:
//     fwd   Y[T,N]  = X[T,K]  . W[N,K]^T          A K-major,  B K-major
//     dgrad dX[T,K] = dY[T,N] . W[N,K]            A K-major,  B MN-major (stored [N(contraction), K(out)])
//     wgrad dW[N,K] = dY[T,N]^T . X[T,K]          A MN-major, B MN-major (contraction over T)
#include <string.h>

#include "common.cuh"
#include "wgmma.cuh"
#include "../../include/dolomite_b200.h"

using namespace dolo;

namespace {

constexpr int BM = 128;
constexpr int BN = 128;  // tile width of the grouped, gather-on-load and split-K modes and of fp8 launches
constexpr int BK = 64;   // bf16 k-block: 64 bf16 = 128 bytes = one swizzle span
constexpr int A_STAGE_BYTES = BM * BK * 2;  // 16 KB
constexpr int GEMM_THREADS = 384;  // warpgroup 0 producer, 1..2 consumers

// Epilogue staging: each consumer warpgroup owns two slabs of 64 rows x 128 B (64 bf16 or 32 fp32
// columns, 128B-swizzled like the D / C tensor maps) and a copy of the tile's bias slice (up to 256 bf16).
constexpr int EPI_SLAB_BYTES = 64 * 128;
constexpr int EPI_BYTES = 2 /*warpgroups*/ * 2 /*slabs*/ * EPI_SLAB_BYTES;
constexpr int EPI_BIAS_BYTES = 2 /*warpgroups*/ * 256 * 2;

// Shared memory of the kernel per output tile width TN: the stage ring (128 x 128 keeps six 32 KB stages, 128 x 256
// four 48 KB stages), then the epilogue slabs, the bias slices and the barriers.
template <int TN>
struct Ring {
    static_assert(TN == 128 || TN == 256, "tile width 128 or 256");
    static constexpr int STAGES = TN == 256 ? 4 : 6;
    static constexpr int B_BYTES = TN * BK * 2;
    static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_BYTES;
    static constexpr int EPI_OFFSET = STAGES * STAGE_BYTES;  // a multiple of 1024: the slabs keep the swizzle alignment
    static constexpr int BIAS_OFFSET = EPI_OFFSET + EPI_BYTES;
    static constexpr int BAR_OFFSET = BIAS_OFFSET + EPI_BIAS_BYTES;
    static constexpr int SMEM_BYTES = 1024 /*align slack*/ + BAR_OFFSET + 256 /*barriers*/;
    static_assert(EPI_OFFSET % 1024 == 0, "epilogue slabs must stay 1024-byte aligned");
    static_assert((2 * STAGES + 4) * 8 <= 256, "barrier area");
    static_assert(SMEM_BYTES <= 232448, "shared memory budget exceeded (227 KB per block on sm_90)");
};

// Registers per thread of the 128 x 256 kernel after setmaxnreg: the producer warpgroup only issues TMA loads, the
// consumers hold 128 fp32 accumulators each.  40 * 128 + 2 * 232 * 128 <= 65536 registers per SM.
constexpr int PRODUCER_REGS = 40;
constexpr int CONSUMER_REGS = 232;
static_assert(PRODUCER_REGS * 128 + 2 * CONSUMER_REGS * 128 <= 65536, "register file exceeded");

// Time of one 128 x 256 tile over one 128 x 128 tile of the same K (see choose_tile_n): the median over the twelve bf16
// GEMM launches of a C2 training step in two passes of tools/bench_gemm.py on an H100 80GB HBM3 at a 400 W power limit
// (per launch 1.26 .. 1.85).  The shared-memory epilogue removed most of the fixed cost per tile, which weighed more on
// the 128 x 256 tile, so the ratio fell from 1.81.  Every value below 5/3 makes the same choice at C2: 256 for every
// launch, including the 4096 x 2560 outputs (3 waves against 5); a whole C2 step confirms that choice.
constexpr double TILE256_COST = 1.65;

constexpr int MAXP = 4;  // problems per launch (the four weight gradients of a transformer block share one launch)

// d / c: rank-3 maps {N, M, groups} of D and C with a box of one epilogue slab {128 B of columns, 64 rows, 1} (the group
// dimension is 1 except for the K-grouped expert weight gradients)
struct GemmMaps {
    CUtensorMap a[MAXP], b[MAXP], d[MAXP], c[MAXP];
};

struct Problem {
    void* D;
    const void* C;
    const __nv_bfloat16* bias;
    int64_t ldd, ldc;
    int M, N;
    int num_m, num_n, num_kb;
    int group_m;     // m-blocks per rasterisation panel
    int tile_start;  // first launch-wide tile index of this problem
    float alpha, beta;
    uint64_t hint_a, hint_b;  // L2 eviction priority of the operand loads (TMA_HINT_*)
};

struct GemmParams {
    Problem pr[MAXP];
    int n_prob;
    int num_tiles;  // over all problems (grouped modes: single problem, includes the group factor)
    int d_is_f32;
    // grouped modes (MoE experts; moe_dolomite/moe/scatter.py:38-49 parallel_linear):
    //   1 = M-grouped: every 128-row tile of A/D belongs to one group (m_tile_group[m_blk], -1 = unused tile); a K-major
    //       B's outer TMA coordinate is offset by group * b_group_rows, an MN-major B's rank-3 map takes the group as its
    //       third coordinate (fwd / dgrad of the expert linears)
    //   2 = K-grouped: tile index also enumerates the group; the contraction runs over rows
    //       [group_k_offsets[g], group_k_offsets[g+1]) and D/C are slice g of their rank-3 maps (expert wgrad)
    int grouped;
    const int* m_tile_group;
    const int* a_row_index;  // gather-on-load: source row of A for every (grouped) row of the problem, or NULL
    const void* gather_a;    // gather-on-load: the ungrouped A [a_rows, K] (row stride gather_lda), read by the producer warp
    int64_t gather_lda;
    int gather_k;
    int b_group_rows;
    const int* group_k_offsets;
    int num_groups;
    int64_t bias_group_stride;  // M-grouped: group g reads its bias row at pr.bias + g * bias_group_stride (0: dense)
    const float* a_scale_inv[MAXP];  // fp8: scale_inv of A and of B per problem (device scalars)
    const float* b_scale_inv[MAXP];
};

struct TileInfo {
    int q;  // problem index
    int m_blk, n_blk, grp, kb0, kb1;
    bool valid;
};

// Tile rasterisation: sweep all n-blocks for a panel of `gm` m-blocks, so that the A panel (gm x 128 rows x K) stays
// L2-resident while B streams; gm is chosen on the host so that the panel is ~12 MB of the 50 MB L2 (with a
// fixed panel of 8, B is re-read 8x from DRAM).
__device__ __forceinline__ void tile_coords(int t, int num_m, int num_n, int gm, int& m_blk, int& n_blk) {
    const int per_group = gm * num_n;
    const int group = t / per_group;
    const int first_m = group * gm;
    const int gsize = min(num_m - first_m, gm);
    const int r = t - group * per_group;
    m_blk = first_m + r % gsize;
    n_blk = r / gsize;
}

// GROUPED: the operand type has the launch modes of p.grouped (otherwise every launch is dense)
template <bool GROUPED>
__device__ __forceinline__ TileInfo tile_info(int t, const GemmParams& p) {
    TileInfo ti;
    ti.q = 0;
#pragma unroll
    for (int i = 1; i < MAXP; ++i)
        if (i < p.n_prob && t >= p.pr[i].tile_start) ti.q = i;
    const Problem& pr = p.pr[ti.q];
    t -= pr.tile_start;
    ti.grp = 0;
    ti.kb0 = 0;
    ti.kb1 = pr.num_kb;
    ti.valid = true;
    if (GROUPED && p.grouped == 3) {
        // split-K: tile index also enumerates the K split; partial products are reduce-added (TMA, fp32)
        const int per = pr.num_m * pr.num_n;
        const int split = t / per;
        tile_coords(t - split * per, pr.num_m, pr.num_n, pr.group_m, ti.m_blk, ti.n_blk);
        const int kb_per = (pr.num_kb + p.num_groups - 1) / p.num_groups;
        ti.kb0 = split * kb_per;
        ti.kb1 = min(pr.num_kb, ti.kb0 + kb_per);
        ti.valid = ti.kb1 > ti.kb0;
    } else if (GROUPED && p.grouped == 2) {
        const int per = pr.num_m * pr.num_n;
        ti.grp = t / per;
        tile_coords(t - ti.grp * per, pr.num_m, pr.num_n, pr.group_m, ti.m_blk, ti.n_blk);
        ti.kb0 = p.group_k_offsets[ti.grp] / BK;
        ti.kb1 = p.group_k_offsets[ti.grp + 1] / BK;
        ti.valid = ti.kb1 > ti.kb0;
    } else {
        tile_coords(t, pr.num_m, pr.num_n, pr.group_m, ti.m_blk, ti.n_blk);
        if (GROUPED && p.grouped == 1) {
            ti.grp = p.m_tile_group[ti.m_blk];
            ti.valid = ti.grp >= 0;
        }
    }
    return ti;
}

// Epilogue state of one consumer warpgroup.  Its 64 rows of the tile leave in chunks of one slab (64 bf16 or 32 fp32
// columns), alternating between its two slabs.  A slab is rewritten only after the store that last read it has finished
// reading.  Chunks 0 and 1 of a tile reuse slabs whose stores were issued before the tile's mainloop (begin_tile), so
// they never wait; chunks 2 and up (128 x 256 bf16, fp32) wait for the store of the chunk two back, while the previous
// chunk's store stays in flight.  The stores of a tile's last chunks run on during the next tile's mainloop.  C, when
// present, is TMA-loaded into the slab that then receives the result: chunks 0 and 1 during the mainloop
// (load_c_prefetch), later ones when their slab comes free.
struct Epilogue {
    uint8_t* slabs;         // [2][EPI_SLAB_BYTES]
    uint32_t* bias;         // [TN / 2] bf16 pairs of the tile's bias slice
    uint64_t* c_bar;        // [2] C arrival per slab
    int slab = 0;           // slab of the next chunk
    uint32_t c_phase = 0;   // bit s: parity of the next wait on c_bar[s]
    int cw;                 // consumer warpgroup: named barrier 1 + cw
    bool leader;            // thread 0 of the warpgroup: issues the TMA traffic and owns its bulk async-groups

    // C of chunks 0 and 1 of the tile (row0, col0), once the previous tile's stores have read both slabs
    __device__ __forceinline__ void load_c_prefetch(const CUtensorMap* cmap, int chunk_cols, int col0, int row0, int grp) {
        tma_store_wait_read<0>();
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int s = slab ^ i;
            mbar_expect_tx(&c_bar[s], EPI_SLAB_BYTES);
            tma_load_3d(slabs + s * EPI_SLAB_BYTES, cmap, &c_bar[s], col0 + i * chunk_cols, row0, grp);
        }
    }

    // after the tile's mainloop: the previous tile's stores have read both slabs (they were issued a mainloop ago), and
    // the barrier also publishes the tile's bias slice
    __device__ __forceinline__ void begin_tile() {
        if (leader) tma_store_wait_read<0>();
        named_bar_sync(1 + cw, 128);
    }

    // chunk ch >= 2 goes to the slab of chunk ch - 2: wait until that chunk's store has read it (the store of chunk
    // ch - 1 may stay in flight); the leader then TMA-loads the chunk's C into it if there is one
    __device__ __forceinline__ void reuse_slab(bool has_c, const CUtensorMap* cmap, int col, int row0, int grp) {
        if (leader) {
            tma_store_wait_read<1>();
            if (has_c) {
                mbar_expect_tx(&c_bar[slab], EPI_SLAB_BYTES);
                tma_load_3d(slabs + slab * EPI_SLAB_BYTES, cmap, &c_bar[slab], col, row0, grp);
            }
        }
        named_bar_sync(1 + cw, 128);
    }

    // D tile (row0, col0) of group grp = (acc + bias) * alpha (+ beta * C), or with SCALED (s * acc + bias) * alpha
    // (+ beta * C), written (or reduce-added) through the slabs.  The fp32 expression and its order are those of a plain
    // register epilogue, so results do not depend on the path.  s stays inside the expression (s * acc + bias contracts
    // to one FFMA), so it is not folded into the accumulators beforehand.
    template <int TN, bool F32, bool SCALED>
    __device__ __forceinline__ void store(const float (&acc)[TN / 2], const CUtensorMap* dmap, const CUtensorMap* cmap,
                                          int col0, int row0, int grp, float s, float alpha, float beta, bool has_bias,
                                          bool has_c, bool reduce) {
        constexpr int CHUNK = F32 ? 32 : 64;  // columns of one slab
        constexpr int NB = CHUNK / 8;         // n8 accumulator blocks per slab
        const int lane = threadIdx.x & 31;
        const int wrow = ((threadIdx.x >> 5) & 3) * 16;  // this warp's first row inside the warpgroup's 64
        auto scaled = [s](float a) { return SCALED ? s * a : a; };
#pragma unroll
        for (int ch = 0; ch < TN / CHUNK; ++ch) {
            uint8_t* sl = slabs + slab * EPI_SLAB_BYTES;
            if (ch >= 2) reuse_slab(has_c, cmap, col0 + ch * CHUNK, row0, grp);
            if (has_c) {
                mbar_wait(&c_bar[slab], (c_phase >> slab) & 1u, 4);
                c_phase ^= 1u << slab;
            }
            if constexpr (F32) {
                // thread: rows lane / 4 (+8) of its warp, columns 2 (lane % 4) (+1) of each n8 block; 128B swizzle:
                // 16-byte unit u of slab row r lives at unit u ^ (r % 8)
#pragma unroll
                for (int jj = 0; jj < NB; ++jj) {
                    const int j = ch * NB + jj;
                    float b0 = 0.f, b1 = 0.f;
                    if (has_bias) {
                        const uint32_t bv = bias[4 * j + (lane & 3)];
                        b0 = bf16_lo(bv);
                        b1 = bf16_hi(bv);
                    }
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int r = wrow + 8 * h + (lane >> 2);
                        const int byte = jj * 32 + (lane & 3) * 8;
                        float2* d = reinterpret_cast<float2*>(sl + r * 128 + ((((byte >> 4) ^ (r & 7)) << 4) | (byte & 15)));
                        float v0 = (scaled(acc[4 * j + 2 * h]) + b0) * alpha;
                        float v1 = (scaled(acc[4 * j + 2 * h + 1]) + b1) * alpha;
                        if (has_c) {
                            const float2 c2 = *d;
                            v0 += beta * c2.x;
                            v1 += beta * c2.y;
                        }
                        *d = make_float2(v0, v1);
                    }
                }
            } else {
                // one x4 matrix move per pair of n8 blocks: matrix m = lane / 8 is n8 block jj + m / 2, rows 8 (m % 2) ..+7
                const int m = lane >> 3;
                const int r = wrow + 8 * (m & 1) + (lane & 7);
#pragma unroll
                for (int jj = 0; jj < NB; jj += 2) {
                    const uint32_t addr = smem_u32(sl + r * 128 + (((jj + (m >> 1)) ^ (lane & 7)) << 4));
                    uint32_t cv[4], out[4];
                    if (has_c) ldmatrix_x4(addr, cv);
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const int j = ch * NB + jj + (i >> 1), h = i & 1;
                        float b0 = 0.f, b1 = 0.f;
                        if (has_bias) {
                            const uint32_t bv = bias[4 * j + (lane & 3)];
                            b0 = bf16_lo(bv);
                            b1 = bf16_hi(bv);
                        }
                        float v0 = (scaled(acc[4 * j + 2 * h]) + b0) * alpha;
                        float v1 = (scaled(acc[4 * j + 2 * h + 1]) + b1) * alpha;
                        if (has_c) {
                            v0 += beta * bf16_lo(cv[i]);
                            v1 += beta * bf16_hi(cv[i]);
                        }
                        out[i] = pack_bf16(v0, v1);
                    }
                    stmatrix_x4(addr, out);
                }
            }
            issue(dmap, col0 + ch * CHUNK, row0, grp, reduce);
        }
    }

    // zero D tile of an fp32 launch, stored from zeroed slabs
    template <int TN>
    __device__ __forceinline__ void store_zero_f32(const CUtensorMap* dmap, int col0, int row0, int grp) {
        begin_tile();
#pragma unroll 1
        for (int ch = 0; ch < TN / 32; ++ch) {
            if (ch >= 2) reuse_slab(false, nullptr, 0, 0, 0);
            uint4* s = reinterpret_cast<uint4*>(slabs + slab * EPI_SLAB_BYTES);
#pragma unroll
            for (int i = 0; i < EPI_SLAB_BYTES / 16 / 128; ++i) s[(threadIdx.x & 127) + 128 * i] = make_uint4(0u, 0u, 0u, 0u);
            issue(dmap, col0 + ch * 32, row0, grp, false);
        }
    }

    // the current slab is written: the leader stores (or reduce-adds) it to the chunk at (col, row0) and moves on to
    // the other slab.  D's tensor map clips the M and N tails.
    __device__ __forceinline__ void issue(const CUtensorMap* dmap, int col, int row0, int grp, bool reduce) {
        const uint8_t* sl = slabs + slab * EPI_SLAB_BYTES;
        fence_proxy_async_smem();  // the slab's writes -> visible to the TMA store (async proxy)
        named_bar_sync(1 + cw, 128);
        if (leader) {
            if (reduce)
                tma_reduce_add_3d(dmap, sl, col, row0, grp);
            else
                tma_store_3d(dmap, sl, col, row0, grp);
            tma_store_commit();
        }
        slab ^= 1;
    }
};

// Operand policies: what differs between the bf16 and the fp8 instances of the kernel body.  A k-block is one 128-byte
// swizzle span of a row in both (64 bf16 or 128 fp8 elements), so the stages, the TMA boxes in bytes and the shared-memory
// descriptors (+32 B per MMA step, four steps per k-block) are the same.
//   KB_ELEMS  elements per k-block (the K coordinate of the TMA loads)
//   mma       one MMA step of a consumer warpgroup: wgmma k16 bf16, or k32 fp8 (K-major operands, 128-wide tile only)
//   SPLIT     promote per k-block: the accumulator is added into a second register set after every k-block and the
//             next k-block starts from zero (TransformerEngine's split accumulator, used for dgrad / wgrad)
//   SCALED    the epilogue has a scale: s = scale_inv_a * scale_inv_b of the problem
//   GROUPED   the launch modes of p.grouped (grouped experts, gather-on-load, split-K) and MN-major operands exist
template <bool A_MN_, bool B_MN_>
struct Bf16Ops {
    static constexpr bool A_MN = A_MN_, B_MN = B_MN_;
    static constexpr int KB_ELEMS = BK;
    static constexpr bool SPLIT = false, SCALED = false, GROUPED = true;
    template <int TN>
    static __device__ __forceinline__ void mma(float (&acc)[TN / 2], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
        wgmma_ss<TN, A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, adesc, bdesc, scale_d);
    }
};

template <int FA, int FB, bool SPLIT_>
struct Fp8Ops {
    static constexpr bool A_MN = false, B_MN = false;
    static constexpr int KB_ELEMS = 128;
    static constexpr bool SPLIT = SPLIT_, SCALED = true, GROUPED = false;
    template <int TN>
    static __device__ __forceinline__ void mma(float (&acc)[TN / 2], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
        static_assert(TN == 128, "fp8 tiles are 128 wide");
        wgmma_fp8_n128<FA, FB>(acc, adesc, bdesc, scale_d);
    }
};

// TN: output tile width.  The 128 x 256 tile runs dense bf16 launches only (grouped == 0, no gather), because the grouped
// modes' tile tables are per 128 x 128 tile.
template <class Op, int TN>
__device__ __forceinline__ void gemm_body(const GemmMaps& maps, const GemmParams& p) {
    constexpr bool A_MN = Op::A_MN, B_MN = Op::B_MN;
    constexpr int STAGES = Ring<TN>::STAGES;
    constexpr int B_STAGE_BYTES = Ring<TN>::B_BYTES;
    constexpr int STAGE_BYTES = Ring<TN>::STAGE_BYTES;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_align_1024(smem_raw);
    uint8_t* smem_a = smem;
    uint8_t* smem_b = smem + STAGES * A_STAGE_BYTES;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Ring<TN>::BAR_OFFSET);
    uint64_t* full_bar = bars;                 // [STAGES]
    uint64_t* empty_bar = bars + STAGES;       // [STAGES]
    uint64_t* c_bar = bars + 2 * STAGES;       // [2 consumer warpgroups][2 slabs]

    const int wg = threadIdx.x >> 7;
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int num_tiles = p.num_tiles;
    const bool gather = Op::GROUPED && TN == 128 && !A_MN && p.a_row_index != nullptr;

    if (threadIdx.x == 0) {
        for (int q = 0; q < p.n_prob; ++q) {
            if (!gather) tma_prefetch_desc(&maps.a[q]);
            tma_prefetch_desc(&maps.b[q]);
        }
        for (int i = 0; i < STAGES; ++i) {
            // gather-on-load: the 32 producer lanes arrive after their shared-memory stores, lane 0 also carries B's bytes
            mbar_init(&full_bar[i], gather ? 33 : 1);
            mbar_init(&empty_bar[i], 8);  // one arrive per consumer warp
        }
        for (int i = 0; i < 4; ++i) mbar_init(&c_bar[i], 1);
        mbar_fence_init();
    }
    __syncthreads();

    if (wg == 0) {
        // ================= producer =================
        if constexpr (TN == 256) setmaxnreg_dec<PRODUCER_REGS>();  // all four warps, before warps 1..3 leave
        if (warp != 0) return;
        if (gather) {
            // Gather-on-load (grouped expert GEMM reading the UNGROUPED activations): lane l copies rows 4l .. 4l+3 of the
            // 128-row A tile from their source rows into the 128B-swizzled stage (16-byte chunk c of row r lands at chunk
            // c ^ (r % 8), the layout TMA would have written); lane 0 also loads B through TMA.
            const __nv_bfloat16* A = static_cast<const __nv_bfloat16*>(p.gather_a);
            int stage = 0;
            uint32_t phase = 0;
            for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
                const TileInfo ti = tile_info<Op::GROUPED>(t, p);
                if (!ti.valid) continue;
                const CUtensorMap* tmap_b = &maps.b[ti.q];
                const int b_outer = ti.grp * p.b_group_rows;
                const int4 src = *reinterpret_cast<const int4*>(p.a_row_index + int64_t(ti.m_blk) * BM + lane * 4);
                const int srow[4] = {src.x, src.y, src.z, src.w};
                for (int kb = ti.kb0; kb < ti.kb1; ++kb) {
                    mbar_wait(&empty_bar[stage], phase ^ 1, 1);
                    uint8_t* sa = smem_a + stage * A_STAGE_BYTES;
                    uint8_t* sb = smem_b + stage * B_STAGE_BYTES;
                    if (lane == 0) {
                        mbar_expect_tx(&full_bar[stage], B_STAGE_BYTES);
                        if (!B_MN) {
                            tma_load_2d(sb, tmap_b, &full_bar[stage], kb * BK, b_outer + ti.n_blk * BN);
                        } else {
#pragma unroll
                            for (int i = 0; i < BN / 64; ++i)
                                tma_load_2d(sb + i * (BK * 128), tmap_b, &full_bar[stage], ti.n_blk * BN + i * 64,
                                            b_outer + kb * BK);
                        }
                    }
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const int r = lane * 4 + i;
                        const __nv_bfloat16* g = A + int64_t(srow[i]) * p.gather_lda + int64_t(kb) * BK;
#pragma unroll
                        for (int c = 0; c < 8; ++c) {
                            uint4 v = make_uint4(0u, 0u, 0u, 0u);
                            if (kb * BK + c * 8 < p.gather_k) v = __ldg(reinterpret_cast<const uint4*>(g + c * 8));
                            *reinterpret_cast<uint4*>(sa + r * 128 + ((c ^ (r & 7)) << 4)) = v;
                        }
                    }
                    fence_proxy_async_smem();  // generic-proxy stores -> visible to wgmma (async proxy)
                    mbar_arrive(&full_bar[stage]);
                    if (++stage == STAGES) { stage = 0; phase ^= 1; }
                }
            }
        } else if (elect_one()) {
            int stage = 0;
            uint32_t phase = 0;
            for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
                const TileInfo ti = tile_info<Op::GROUPED>(t, p);
                if (!ti.valid) continue;
                const CUtensorMap* tmap_a = &maps.a[ti.q];
                const CUtensorMap* tmap_b = &maps.b[ti.q];
                const uint64_t ha = p.pr[ti.q].hint_a, hb = p.pr[ti.q].hint_b;
                const int m_blk = ti.m_blk, n_blk = ti.n_blk;
                const int b_outer = (Op::GROUPED && p.grouped == 1 && !B_MN) ? ti.grp * p.b_group_rows : 0;
                for (int kb = ti.kb0; kb < ti.kb1; ++kb) {
                    mbar_wait(&empty_bar[stage], phase ^ 1, 1);
                    uint8_t* sa = smem_a + stage * A_STAGE_BYTES;
                    uint8_t* sb = smem_b + stage * B_STAGE_BYTES;
                    mbar_expect_tx(&full_bar[stage], STAGE_BYTES);
                    if (!A_MN) {
                        tma_load_2d_hint(sa, tmap_a, &full_bar[stage], kb * Op::KB_ELEMS, m_blk * BM, ha);
                    } else {
#pragma unroll
                        for (int i = 0; i < BM / 64; ++i)
                            tma_load_2d_hint(sa + i * (BK * 128), tmap_a, &full_bar[stage], m_blk * BM + i * 64, kb * BK, ha);
                    }
                    if (!B_MN) {
                        tma_load_2d_hint(sb, tmap_b, &full_bar[stage], kb * Op::KB_ELEMS, b_outer + n_blk * TN, hb);
                    } else if (Op::GROUPED && p.grouped == 1) {
                        // M-grouped dgrad: B's rank-3 map {N, K, groups} zero-fills the K tail of the tile's own expert
                        // (grouped launches load with the normal L2 priority, so no hint)
#pragma unroll
                        for (int i = 0; i < TN / 64; ++i)
                            tma_load_3d(sb + i * (BK * 128), tmap_b, &full_bar[stage], n_blk * TN + i * 64, kb * BK, ti.grp);
                    } else {
#pragma unroll
                        for (int i = 0; i < TN / 64; ++i)
                            tma_load_2d_hint(sb + i * (BK * 128), tmap_b, &full_bar[stage], n_blk * TN + i * 64,
                                             b_outer + kb * BK, hb);
                    }
                    if (++stage == STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
        return;
    }

    // ================= consumers: warpgroup cw owns rows [64 cw, 64 cw + 64) of the tile =================
    if constexpr (TN == 256) setmaxnreg_inc<CONSUMER_REGS>();
    const int cw = wg - 1;
    const int wt = threadIdx.x & 127;  // thread inside the warpgroup
    Epilogue epi;
    epi.slabs = smem + Ring<TN>::EPI_OFFSET + cw * 2 * EPI_SLAB_BYTES;
    epi.bias = reinterpret_cast<uint32_t*>(smem + Ring<TN>::BIAS_OFFSET + cw * (EPI_BIAS_BYTES / 2));
    epi.c_bar = c_bar + 2 * cw;
    epi.cw = cw;
    epi.leader = wt == 0;
    const int chunk_cols = p.d_is_f32 ? 32 : 64;
    int stage = 0;
    uint32_t phase = 0;
    float acc[TN / 2];
    float tot[TN / 2];  // SPLIT: the sum of the promoted k-blocks
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        const TileInfo ti = tile_info<Op::GROUPED>(t, p);
        const Problem& pr = p.pr[ti.q];
        const int row0 = ti.m_blk * BM + cw * 64;  // first row of this warpgroup's 64
        const int col0 = ti.n_blk * TN;
        const int dgrp = Op::GROUPED && p.grouped == 2 ? ti.grp : 0;
        // K-grouped launch (expert weight gradients) and this expert received NO rows: its product is zero.  A launch that
        // OVERWRITES (beta = 0, no C) must still write the tile -- the caller did not clear the buffer.
        if (!ti.valid) {
            if (Op::GROUPED && p.grouped == 2 && p.d_is_f32 && pr.C == nullptr) epi.store_zero_f32<TN>(&maps.d[ti.q], col0, row0, dgrp);
            continue;
        }
        const bool has_bias = pr.bias != nullptr;
        const bool has_c = pr.C != nullptr;
        // the tile's bias slice (of the tile's group's bias row in the M-grouped mode): loaded now, kept in shared memory
        // for the epilogue.  An odd N ends in a half pair, whose upper element (column N) is not read; its value only ever
        // reaches the clipped column N of the slab.
        uint32_t bias_v = 0;
        if (has_bias && wt < TN / 2 && col0 + 2 * wt < pr.N) {
            const __nv_bfloat16* brow = pr.bias + ti.grp * p.bias_group_stride;
            if (col0 + 2 * wt + 1 < pr.N)
                bias_v = __ldg(reinterpret_cast<const uint32_t*>(brow + col0 + 2 * wt));
            else
                bias_v = __bfloat16_as_ushort(brow[col0 + 2 * wt]);
        }
        int prev_stage = -1;
        for (int kb = ti.kb0; kb < ti.kb1; ++kb) {
            mbar_wait(&full_bar[stage], phase, 3);
            wgmma_fence();
            const uint32_t sa = smem_u32(smem_a + stage * A_STAGE_BYTES);
            const uint32_t sb = smem_u32(smem_b + stage * B_STAGE_BYTES);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                // K-major: +32 B per MMA step (K=16 bf16, K=32 fp8) inside the 128 B swizzle span; SBO = 8 rows x 128 B;
                // this warpgroup's 64 rows start 64 x 128 B into the tile.
                // MN-major: +16 K-rows x 128 B per step; LBO = next 64-wide MN chunk (BK rows x 128 B), SBO = 8 K-rows;
                // this warpgroup's 64 rows are the cw-th chunk.
                const uint64_t adesc = A_MN ? gmma_desc(sa + cw * (BK * 128) + k * 2048, BK * 128, 1024, 1)
                                            : gmma_desc(sa + cw * (64 * 128) + k * 32, 16, 1024, 1);
                const uint64_t bdesc = B_MN ? gmma_desc(sb + k * 2048, BK * 128, 1024, 1)
                                            : gmma_desc(sb + k * 32, 16, 1024, 1);
                Op::template mma<TN>(acc, adesc, bdesc, ((!Op::SPLIT && kb != ti.kb0) || k != 0) ? 1u : 0u);
            }
            wgmma_commit();
            // C of the tile's first two chunks: the load overlaps the rest of the mainloop.  Two k-blocks in, the
            // previous tile's last stores have long read their slabs, so the leader does not hold up the MMAs.
            if (kb == min(ti.kb0 + 2, ti.kb1 - 1) && has_c && epi.leader) epi.load_c_prefetch(&maps.c[ti.q], chunk_cols, col0, row0, dgrp);
            if constexpr (Op::SPLIT) {
                wgmma_wait<0>();  // this k-block's MMAs retired: its stage may be refilled, its product promoted
                reg_fence<TN / 2>(acc);
                if (lane == 0) mbar_arrive(&empty_bar[stage]);
                if (kb == ti.kb0) {
#pragma unroll
                    for (int i = 0; i < TN / 2; ++i) tot[i] = acc[i];
                } else {
#pragma unroll
                    for (int i = 0; i < TN / 2; ++i) tot[i] += acc[i];
                }
            } else {
                wgmma_wait<1>();  // the previous k-block's MMAs retired: its stage may be refilled
                if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);
                prev_stage = stage;
            }
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
        if constexpr (!Op::SPLIT) {
            wgmma_wait<0>();
            reg_fence<TN / 2>(acc);
            if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);
        }
        const float(&res)[TN / 2] = Op::SPLIT ? tot : acc;
        float s = 1.f;
        if constexpr (Op::SCALED) s = __ldg(p.a_scale_inv[ti.q]) * __ldg(p.b_scale_inv[ti.q]);
        // the previous tile's epilogue has finished reading the bias slice: its last chunk ended in a barrier
        if (has_bias && wt < TN / 2) epi.bias[wt] = bias_v;
        epi.begin_tile();

        // ---------------- epilogue: registers -> shared-memory slabs -> TMA ----------------
        if (p.d_is_f32)
            epi.store<TN, true, Op::SCALED>(res, &maps.d[ti.q], &maps.c[ti.q], col0, row0, dgrp, s, pr.alpha, pr.beta,
                                            has_bias, has_c, Op::GROUPED && p.grouped == 3);
        else
            epi.store<TN, false, Op::SCALED>(res, &maps.d[ti.q], &maps.c[ti.q], col0, row0, dgrp, s, pr.alpha, pr.beta,
                                             has_bias, has_c, false);
    }
    if (epi.leader) tma_store_wait_all<0>();  // the slabs must outlive the stores that read them
}

template <bool A_MN, bool B_MN, int TN>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
    gemm_bf16_kernel(const __grid_constant__ GemmMaps maps, const __grid_constant__ GemmParams p) {
    gemm_body<Bf16Ops<A_MN, B_MN>, TN>(maps, p);
}

// FP8 GEMM (TransformerEngine te.Linear under fp8_autocast): A [M, K] and B [N, K] are both row-major (the transposes come
// from the cast kernel), 128 x 128 tiles.
//   D = alpha * (scale_inv_a * scale_inv_b * acc + bias) + beta * C
// SPLIT: split accumulation (dgrad / wgrad); otherwise the MMA accumulates over the whole contraction (fprop, TE's fast
// accumulation).
template <int FA, int FB, bool SPLIT>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
    gemm_fp8_kernel(const __grid_constant__ GemmMaps maps, const __grid_constant__ GemmParams p) {
    gemm_body<Fp8Ops<FA, FB, SPLIT>, 128>(maps, p);
}

// SMs of the static persistent schedule: worker w takes tiles w, w + W, ... on `SMs - gemm_sm_margin` SMs
int gemm_workers() {
    const int sms = dolo_num_sms() - dolo_option_gemm_sm_margin();
    return sms < 1 ? 1 : sms;
}

template <int TN, void (*KERNEL)(GemmMaps, GemmParams)>
int launch_gemm(const GemmMaps& maps, const GemmParams& p, cudaStream_t st) {
    constexpr int smem_bytes = Ring<TN>::SMEM_BYTES;
    static bool attr_set = false;  // per instantiation
    if (!attr_set) {
        DOLO_CUDA_OK(cudaFuncSetAttribute(KERNEL, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
        attr_set = true;
    }
    const int sms = gemm_workers();
    const int grid = p.num_tiles < sms ? p.num_tiles : sms;
    KERNEL<<<grid, GEMM_THREADS, smem_bytes, st>>>(maps, p);
    DOLO_LAUNCH_OK("gemm");
    return DOLO_OK;
}

// Tile width of a dense launch.  The static persistent schedule gives its busiest worker ceil(tiles / workers) tiles, so
// a launch costs ceil(tiles_w / workers) * c_w.  The 128 x 256 tile moves 25 % fewer operand bytes per FLOP and runs
// closer to the tensor-core peak (TILE256_COST < 2), but halves the tile count: where it leaves a partly filled last wave
// that the 128 x 128 tiles fill, the narrow tile can win (a 4096 x 2560 output: 4.85 waves of 128-wide tiles on 132 SMs,
// 2.42 of 256-wide ones, so 128 wins iff TILE256_COST > 5/3).
int choose_tile_n(int n, const int64_t* M, const int64_t* N) {
    const int forced = dolo_option_gemm_tile_n();
    if (forced != 0) return forced;
    const int64_t w = gemm_workers();
    int64_t t128 = 0, t256 = 0;
    for (int q = 0; q < n; ++q) {
        const int64_t mb = (M[q] + BM - 1) / BM;
        t128 += mb * ((N[q] + 127) / 128);
        t256 += mb * ((N[q] + 255) / 256);
    }
    const double c128 = double((t128 + w - 1) / w);
    const double c256 = double((t256 + w - 1) / w) * TILE256_COST;
    return c256 < c128 ? 256 : 128;
}

}  // namespace

struct GroupArgs {
    int mode = 0;
    const int* a_row_index = nullptr;  // mode 1 only: gather the rows of A on load (A is the ungrouped matrix of a_rows rows)
    int64_t a_rows = 0;
    const int* m_tile_group = nullptr;
    int64_t b_group_rows = 0;   // mode 1, K-major B: rows of one group's B
    const int* group_k_offsets = nullptr;
    int num_groups = 1;
    int64_t d_group_stride = 0;
    int64_t b_total_outer = 0;  // mode 1, K-major B: rows of B's outer TMA dimension over all groups
    int64_t bias_group_stride = 0;  // mode 1 with bias: elements between the bias rows of consecutive groups
};

// one problem of a launch
struct GemmProblemArgs {
    const void* A; int64_t lda;
    const void* B; int64_t ldb;
    void* D; int64_t ldd;
    const void* C; int64_t ldc;
    const void* bias;
    float alpha, beta;
    int64_t M, N, K;
    const float* a_scale_inv = nullptr;  // fp8 operands: their scale_inv (device scalars)
    const float* b_scale_inv = nullptr;
};

// Fills maps.{a,b}[q] and p.pr[q] for one problem.  All problems of a launch share the operand type (ab: bytes per
// element of A and B, 2 = bf16, 1 = fp8), the operand layouts, the output type and the tile width tile_n (128 or 256).
static int setup_problem(GemmMaps& maps, GemmParams& p, int q, const GemmProblemArgs& g, int ab, int a_mn_major,
                         int b_mn_major, int d_is_f32, const GroupArgs& ga, int tile_n) {
    const int64_t M = g.M, N = g.N, K = g.K;
    if (ab == 1) {
        // fp8: K-major operands; N % 16 == 0 keeps every row of D a whole number of 16-byte segments
        DOLO_REQUIRE(M > 0 && N > 0 && K > 0, "gemm_fp8: empty problem (M=%lld N=%lld K=%lld)", (long long)M,
                     (long long)N, (long long)K);
        DOLO_REQUIRE(K % 16 == 0 && N % 16 == 0, "gemm_fp8: K=%lld and N=%lld must be multiples of 16", (long long)K,
                     (long long)N);
        DOLO_REQUIRE(g.lda % 16 == 0 && g.ldb % 16 == 0 && g.lda >= K && g.ldb >= K,
                     "gemm_fp8: lda / ldb must be >= K and multiples of 16 (16-byte aligned fp8 rows)");
        DOLO_REQUIRE(g.a_scale_inv != nullptr && g.b_scale_inv != nullptr, "gemm_fp8: missing scale_inv pointer");
        p.a_scale_inv[q] = g.a_scale_inv;
        p.b_scale_inv[q] = g.b_scale_inv;
    }
    // M, N and K may take any value: the tensor maps carry the exact extents, so TMA zero-fills the operand tails of the
    // last k-block and tile and clips the D rows and columns.  Only the row strides and the base addresses (checked when
    // the tensor maps are made) need 16-byte alignment.  A TMA store writes whole 16-byte segments: when a row of D ends
    // inside one (N not a multiple of 16 bytes), the rest of that segment, columns [N, round_up(N, 16 bytes)), receives
    // zeros, so ldd must cover it.
    DOLO_REQUIRE(K > 0, "gemm: K must be > 0");
    DOLO_REQUIRE(g.lda * ab % 16 == 0 && g.ldb * ab % 16 == 0 && g.ldd % (d_is_f32 ? 4 : 8) == 0,
                 "gemm: leading dimensions must keep 16-byte alignment");
    {
        const int64_t per = d_is_f32 ? 4 : 8;
        DOLO_REQUIRE(g.ldd >= (N + per - 1) / per * per,
                     "gemm: ldd=%lld must cover N=%lld rounded up to 16 bytes (the TMA store writes that segment)",
                     (long long)g.ldd, (long long)N);
    }
    DOLO_REQUIRE(g.C == nullptr || g.ldc % (d_is_f32 ? 4 : 8) == 0, "gemm: ldc alignment");
    DOLO_REQUIRE((reinterpret_cast<uintptr_t>(g.bias) & 3) == 0, "gemm: bias must be 4-byte aligned");
    DOLO_REQUIRE(M < (1ll << 31) && N < (1ll << 31) && K < (1ll << 31), "gemm: dimension too large");
    // K-major: dims {K, rows}, box {one 128-byte k-block, tile rows} (128 for A, tile_n for B).  MN-major (bf16): dims
    // {rows, K}, box {64, 64}.
    uint64_t dims[2], strides[2];
    uint32_t box[2];
    int rc;
    if (ga.a_row_index != nullptr) {
        // gather-on-load: the producer warp reads A's rows itself (no tensor map)
        DOLO_REQUIRE(!a_mn_major, "gemm: gather-on-load needs a K-major A");
        DOLO_REQUIRE((reinterpret_cast<uintptr_t>(g.A) & 15) == 0, "gemm: gather-on-load needs a 16-byte aligned A");
        // the producer warp copies whole 16-byte vectors of a row: a K tail inside a vector would be read as data
        DOLO_REQUIRE(K % 8 == 0, "gemm: gather-on-load needs K %% 8 == 0 (K=%lld)", (long long)K);
        p.gather_a = g.A;
        p.gather_lda = g.lda;
        p.gather_k = int(K);
    } else {
        if (!a_mn_major) {
            dims[0] = uint64_t(K); dims[1] = uint64_t(M); strides[0] = ab; strides[1] = uint64_t(g.lda) * ab;
            box[0] = 128 / ab; box[1] = BM;
        } else {
            dims[0] = uint64_t(M); dims[1] = uint64_t(K); strides[0] = 2; strides[1] = uint64_t(g.lda) * 2;
            box[0] = 64; box[1] = BK;
        }
        rc = dolo_make_tmap(&maps.a[q], g.A, ab, 2, dims, strides, box, DOLO_SW_128);
        if (rc) return rc;
    }
    strides[0] = ab;
    if (!b_mn_major) {
        // M-grouped: the experts' [N, K] matrices stacked into one [groups * N, K]; an N tail of expert g reads rows of
        // expert g + 1, which only reach the clipped output columns >= N
        dims[0] = uint64_t(K); dims[1] = uint64_t(ga.mode == 1 ? ga.b_total_outer : N); strides[1] = uint64_t(g.ldb) * ab;
        box[0] = 128 / ab; box[1] = uint32_t(tile_n);
        rc = dolo_make_tmap(&maps.b[q], g.B, ab, 2, dims, strides, box, DOLO_SW_128);
    } else if (ga.mode == 1) {
        // M-grouped, MN-major: dims {N, K, groups}, box {64, 64, 1}.  Expert g's contraction ends at its own row K, so the
        // K tail of its last k-block is zero-filled rather than read from expert g + 1 (whose rows, multiplied by A's
        // zero-filled columns, would turn a non-finite weight into NaN).
        const uint64_t dims3[3] = {uint64_t(N), uint64_t(K), uint64_t(ga.num_groups)};
        const uint64_t strides3[3] = {2, uint64_t(g.ldb) * 2, uint64_t(K * g.ldb) * 2};
        const uint32_t box3[3] = {64, BK, 1};
        rc = dolo_make_tmap(&maps.b[q], g.B, ab, 3, dims3, strides3, box3, DOLO_SW_128);
    } else {
        dims[0] = uint64_t(N); dims[1] = uint64_t(K); strides[1] = uint64_t(g.ldb) * 2;
        box[0] = 64; box[1] = BK;
        rc = dolo_make_tmap(&maps.b[q], g.B, ab, 2, dims, strides, box, DOLO_SW_128);
    }
    if (rc) return rc;
    {
        // D and C: dims {N, M, groups}, box = one epilogue slab {128 B of columns, 64 rows, 1}
        const uint64_t eb = d_is_f32 ? 4 : 2;
        const int64_t groups = ga.mode == 2 ? ga.num_groups : 1;
        const int64_t group_stride = ga.mode == 2 ? ga.d_group_stride : M * g.ldd;
        uint64_t ddims[3] = {uint64_t(N), uint64_t(M), uint64_t(groups)};
        uint64_t dstrides[3] = {eb, uint64_t(g.ldd) * eb, uint64_t(group_stride) * eb};
        const uint32_t dbox[3] = {uint32_t(128 / eb), 64, 1};
        rc = dolo_make_tmap(&maps.d[q], g.D, int(eb), 3, ddims, dstrides, dbox, DOLO_SW_128);
        if (rc) return rc;
        if (g.C != nullptr) {
            // C: D's dims with C's row stride (the K-grouped mode passes C == D)
            dstrides[1] = uint64_t(g.ldc) * eb;
            if (ga.mode != 2) dstrides[2] = uint64_t(M * g.ldc) * eb;
            rc = dolo_make_tmap(&maps.c[q], g.C, int(eb), 3, ddims, dstrides, dbox, DOLO_SW_128);
            if (rc) return rc;
        }
    }
    Problem& pr = p.pr[q];
    pr.D = g.D;
    pr.C = g.C;
    pr.bias = static_cast<const __nv_bfloat16*>(g.bias);
    pr.ldd = g.ldd;
    pr.ldc = g.ldc;
    pr.M = int(M);
    pr.N = int(N);
    pr.alpha = g.alpha;
    pr.beta = g.C ? g.beta : 0.f;
    pr.hint_a = pr.hint_b = TMA_HINT_NORMAL;
    if (ab == 2 && dolo_option_gemm_l2_hints() && ga.mode == 0 && K >= 4096 && (M + N) * K * 2 > (24ll << 20)) {
        // long contraction, operands larger than what the L2 keeps anyway: stream the bigger one, keep the smaller one
        const bool a_smaller = M <= N;
        pr.hint_a = a_smaller ? TMA_HINT_EVICT_LAST : TMA_HINT_EVICT_FIRST;
        pr.hint_b = a_smaller ? TMA_HINT_EVICT_FIRST : TMA_HINT_EVICT_LAST;
    }
    pr.num_m = int((M + BM - 1) / BM);
    pr.num_n = int((N + tile_n - 1) / tile_n);
    pr.num_kb = int((K * ab + 127) / 128);  // 128-byte k-blocks
    {
        // A panel of group_m x 128 rows x K should fit comfortably in the 50 MB L2 next to the streaming B tiles
        const int64_t panel_bytes = int64_t(BM) * K * ab;
        int64_t gm = (12ll << 20) / (panel_bytes > 0 ? panel_bytes : 1);
        if (gm < 4) gm = 4;
        if (gm > 64) gm = 64;
        pr.group_m = int(gm);
    }
    return DOLO_OK;
}

template <int TN>
static int dispatch_layout(int a_mn_major, int b_mn_major, const GemmMaps& maps, const GemmParams& p, cudaStream_t st) {
    if (!a_mn_major && !b_mn_major) return launch_gemm<TN, gemm_bf16_kernel<false, false, TN>>(maps, p, st);
    if (!a_mn_major && b_mn_major) return launch_gemm<TN, gemm_bf16_kernel<false, true, TN>>(maps, p, st);
    if (a_mn_major && !b_mn_major) return launch_gemm<TN, gemm_bf16_kernel<true, false, TN>>(maps, p, st);
    return launch_gemm<TN, gemm_bf16_kernel<true, true, TN>>(maps, p, st);
}

static int dispatch(int tile_n, int a_mn_major, int b_mn_major, const GemmMaps& maps, const GemmParams& p, cudaStream_t st) {
    return tile_n == 256 ? dispatch_layout<256>(a_mn_major, b_mn_major, maps, p, st)
                         : dispatch_layout<128>(a_mn_major, b_mn_major, maps, p, st);
}

template <int FA, int FB>
static int dispatch_fp8_split(int split, const GemmMaps& maps, const GemmParams& p, cudaStream_t st) {
    return split ? launch_gemm<BN, gemm_fp8_kernel<FA, FB, true>>(maps, p, st)
                 : launch_gemm<BN, gemm_fp8_kernel<FA, FB, false>>(maps, p, st);
}

static int dispatch_fp8(int a_fmt, int b_fmt, int split, const GemmMaps& maps, const GemmParams& p, cudaStream_t st) {
    if (a_fmt == 0 && b_fmt == 0) return dispatch_fp8_split<0, 0>(split, maps, p, st);
    if (a_fmt == 0 && b_fmt == 1) return dispatch_fp8_split<0, 1>(split, maps, p, st);
    if (a_fmt == 1 && b_fmt == 0) return dispatch_fp8_split<1, 0>(split, maps, p, st);
    return dispatch_fp8_split<1, 1>(split, maps, p, st);
}

static int gemm_impl(const void* A, int64_t lda, int a_mn_major, const void* B, int64_t ldb, int b_mn_major, void* D,
                     int64_t ldd, int d_is_f32, const void* C, int64_t ldc, float alpha, float beta, const void* bias,
                     int64_t M, int64_t N, int64_t K, int flags, void* stream, const GroupArgs& ga) {
    DOLO_REQUIRE(M >= 0 && N >= 0 && K >= 0, "gemm: negative dimension");
    if (M == 0 || N == 0) return DOLO_OK;
    const bool tma_store = (flags & DOLO_GEMM_FLAG_TMA_STORE) != 0;
    DOLO_REQUIRE(!tma_store || (!d_is_f32 && C == nullptr), "gemm: TMA-store epilogue needs bf16 D and no C");
    const int tile_n = ga.mode == 0 ? choose_tile_n(1, &M, &N) : BN;
    GemmMaps maps;
    GemmParams p;
    memset(&p, 0, sizeof(p));
    GemmProblemArgs g{A, lda, B, ldb, D, ldd, C, ldc, bias, alpha, beta, M, N, K};
    int rc = setup_problem(maps, p, 0, g, 2, a_mn_major, b_mn_major, d_is_f32, ga, tile_n);
    if (rc) return rc;
    p.n_prob = 1;
    p.pr[0].tile_start = 0;
    p.num_tiles = p.pr[0].num_m * p.pr[0].num_n * (ga.mode >= 2 ? ga.num_groups : 1);
    p.d_is_f32 = d_is_f32;
    p.grouped = ga.mode;
    p.m_tile_group = ga.m_tile_group;
    p.a_row_index = ga.a_row_index;
    p.b_group_rows = int(ga.b_group_rows);
    p.group_k_offsets = ga.group_k_offsets;
    p.num_groups = ga.num_groups;
    p.bias_group_stride = ga.bias_group_stride;
    return dispatch(tile_n, a_mn_major, b_mn_major, maps, p, static_cast<cudaStream_t>(stream));
}

// The weight gradients of one transformer block in ONE persistent launch (autograd of linear.py:5-25 for c_attn, attention
// c_proj, c_fc and mlp c_proj): dW_i[M_i, N_i] (+)= alpha_i * dY_i^T X_i with dY_i [K, M_i], X_i [K, N_i] row-major
// activations (both operands MN-major).  Launched one by one these GEMMs lose to wave quantisation on the last,
// partly filled wave of each; together the tail is paid once.
extern "C" int dolomite_b200_gemm_bf16_wgrad_multi(int n_problems, const void* const* dY, const int64_t* ld_dy,
                                                   const void* const* X, const int64_t* ld_x, float* const* dW,
                                                   const int64_t* ld_dw, const int64_t* M, const int64_t* N, int64_t K,
                                                   const float* alpha, const int* accumulate, void* stream) {
    DOLO_REQUIRE(n_problems >= 1 && n_problems <= MAXP, "wgrad_multi: between 1 and %d problems per launch", MAXP);
    for (int q = 0; q < n_problems; ++q) DOLO_REQUIRE(M[q] > 0 && N[q] > 0, "wgrad_multi: empty problem %d", q);
    const int tile_n = choose_tile_n(n_problems, M, N);
    GemmMaps maps;
    GemmParams p;
    memset(&p, 0, sizeof(p));
    int tiles = 0;
    for (int q = 0; q < n_problems; ++q) {
        GemmProblemArgs g{dY[q], ld_dy[q], X[q], ld_x[q], dW[q], ld_dw[q], accumulate[q] ? dW[q] : nullptr, ld_dw[q], nullptr,
                          alpha[q], 1.f, M[q], N[q], K};
        int rc = setup_problem(maps, p, q, g, 2, 1, 1, 1, GroupArgs(), tile_n);
        if (rc) return rc;
        p.pr[q].tile_start = tiles;
        tiles += p.pr[q].num_m * p.pr[q].num_n;
    }
    p.n_prob = n_problems;
    p.num_tiles = tiles;
    p.d_is_f32 = 1;
    p.grouped = 0;
    p.num_groups = 1;
    return dispatch(tile_n, 1, 1, maps, p, static_cast<cudaStream_t>(stream));
}

extern "C" int dolomite_b200_gemm_bf16_tile_n(int n_problems, const int64_t* M, const int64_t* N, int* tile_n,
                                              float* cost_256_over_128) {
    DOLO_REQUIRE(n_problems >= 1 && n_problems <= MAXP && M != nullptr && N != nullptr && tile_n != nullptr,
                 "gemm_bf16_tile_n: between 1 and %d problems, non-null M, N and tile_n", MAXP);
    *tile_n = choose_tile_n(n_problems, M, N);
    if (cost_256_over_128 != nullptr) *cost_256_over_128 = float(TILE256_COST);
    return DOLO_OK;
}

extern "C" int dolomite_b200_gemm_bf16(const void* A, int64_t lda, int a_mn_major, const void* B, int64_t ldb,
                                       int b_mn_major, void* D, int64_t ldd, int d_is_f32, const void* C, int64_t ldc,
                                       float alpha, float beta, const void* bias, int64_t M, int64_t N, int64_t K,
                                       int flags, void* stream) {
    if (flags & DOLO_GEMM_FLAG_SPLITK_ACCUMULATE) {
        // D(fp32) += alpha * A B^T with the contraction split over several CTAs (TMA fp32 reduce-adds): removes the
        // wave-quantisation tail of weight-gradient GEMMs (few output tiles, long K) and the read of C
        DOLO_REQUIRE(d_is_f32 && bias == nullptr && (C == nullptr || (C == D && beta == 1.f)),
                     "gemm: split-K accumulate needs fp32 D, no bias and C == D with beta == 1");
        const int64_t tiles = ((M + BM - 1) / BM) * ((N + BN - 1) / BN);
        const int64_t num_kb = (K + BK - 1) / BK;
        const int sms = dolo_num_sms();
        int best_s = 1;
        double best = 1e30;
        for (int s = 1; s <= 16; ++s) {
            if (s > 1 && num_kb / s < 8) break;
            const double waves = double((tiles * s + sms - 1) / sms) / double(s);  // in units of one full-K tile time
            if (waves < best - 1e-9) { best = waves; best_s = s; }
        }
        GroupArgs ga;
        ga.mode = 3;
        ga.num_groups = best_s;
        return gemm_impl(A, lda, a_mn_major, B, ldb, b_mn_major, D, ldd, 1, nullptr, 0, alpha, 0.f, nullptr, M, N, K, 0,
                         stream, ga);
    }
    return gemm_impl(A, lda, a_mn_major, B, ldb, b_mn_major, D, ldd, d_is_f32, C, ldc, alpha, beta, bias, M, N, K, flags,
                     stream, GroupArgs());
}

// M-grouped expert GEMM (fwd / dgrad of the expert linears), with the gather fused into the operand load when a_row_index
// is given (A is then the UNGROUPED activation matrix [a_rows, K] and a_row_index[r] names the source row of grouped row r;
// padding rows may name any valid row: their products are never read), and with a per-group bias row
// bias[g * ld_bias .. + N) added to group g's rows when bias is given.
static int grouped_m_impl(const void* A, int64_t lda, int64_t a_rows, const int32_t* a_row_index, const void* B,
                          int64_t ldb, int b_mn_major, void* D, int64_t ldd, const void* bias, int64_t ld_bias,
                          float alpha, int64_t M_max, int64_t N, int64_t K, const int32_t* m_tile_group, int num_groups,
                          int flags, void* stream) {
    DOLO_REQUIRE(M_max % BM == 0, "grouped gemm: M_max=%lld must be a multiple of %d (padded expert segments)",
                 (long long)M_max, BM);
    // MN-major B: the experts' [K, N] matrices follow each other, so K % 8 == 0 keeps every expert's base 16-byte aligned
    DOLO_REQUIRE(!b_mn_major || K % 8 == 0, "grouped gemm: MN-major B needs K %% 8 == 0 (K=%lld)", (long long)K);
    DOLO_REQUIRE(m_tile_group != nullptr && num_groups > 0, "grouped gemm: missing group table");
    if (a_row_index != nullptr) {
        DOLO_REQUIRE(!b_mn_major && a_rows > 0, "grouped gemm (gather): K-major B and a_rows > 0 needed");
        DOLO_REQUIRE((reinterpret_cast<uintptr_t>(a_row_index) & 15) == 0,
                     "grouped gemm (gather): row index must be 16-byte aligned");
    }
    // every group's bias row must keep the 4-byte alignment of the epilogue's paired loads
    DOLO_REQUIRE(bias == nullptr || (ld_bias >= N && ld_bias % 2 == 0),
                 "grouped gemm: ld_bias=%lld must be even and >= N=%lld", (long long)ld_bias, (long long)N);
    GroupArgs ga;
    ga.mode = 1;
    ga.a_row_index = a_row_index;
    ga.a_rows = a_rows;
    ga.m_tile_group = m_tile_group;
    ga.num_groups = num_groups;
    ga.b_group_rows = N;  // K-major B only (an MN-major B has a rank-3 map with one slice per group)
    ga.b_total_outer = N * num_groups;
    ga.bias_group_stride = bias != nullptr ? ld_bias : 0;
    return gemm_impl(A, lda, 0, B, ldb, b_mn_major, D, ldd, 0, nullptr, 0, alpha, 0.f, bias, M_max, N, K, flags, stream,
                     ga);
}

extern "C" int dolomite_b200_gemm_bf16_grouped_m(const void* A, int64_t lda, const void* B, int64_t ldb, int b_mn_major,
                                                 void* D, int64_t ldd, float alpha, int64_t M_max, int64_t N, int64_t K,
                                                 const int32_t* m_tile_group, int num_groups, int flags, void* stream) {
    return grouped_m_impl(A, lda, 0, nullptr, B, ldb, b_mn_major, D, ldd, nullptr, 0, alpha, M_max, N, K, m_tile_group,
                          num_groups, flags, stream);
}

// Same, with the ScatterMoE gather fused into the operand load
extern "C" int dolomite_b200_gemm_bf16_grouped_m_gather(const void* A, int64_t lda, int64_t a_rows,
                                                        const int32_t* a_row_index, const void* B, int64_t ldb, void* D,
                                                        int64_t ldd, float alpha, int64_t M_max, int64_t N, int64_t K,
                                                        const int32_t* m_tile_group, int num_groups, int flags,
                                                        void* stream) {
    DOLO_REQUIRE(a_row_index != nullptr, "grouped gemm (gather): missing row index");
    return grouped_m_impl(A, lda, a_rows, a_row_index, B, ldb, 0, D, ldd, nullptr, 0, alpha, M_max, N, K, m_tile_group,
                          num_groups, flags, stream);
}

// Expert linears with bias (moe/base.py:12-50 ParameterizedExperts with add_bias): D = (A W[g]^T + bias[g]) * alpha, plain
// (a_row_index NULL) or gather-on-load
extern "C" int dolomite_b200_gemm_bf16_grouped_m_bias(const void* A, int64_t lda, int64_t a_rows,
                                                      const int32_t* a_row_index, const void* B, int64_t ldb,
                                                      int b_mn_major, void* D, int64_t ldd, const void* bias,
                                                      int64_t ld_bias, float alpha, int64_t M_max, int64_t N, int64_t K,
                                                      const int32_t* m_tile_group, int num_groups, int flags,
                                                      void* stream) {
    DOLO_REQUIRE(bias != nullptr, "grouped gemm (bias): missing bias");
    return grouped_m_impl(A, lda, a_rows, a_row_index, B, ldb, b_mn_major, D, ldd, bias, ld_bias, alpha, M_max, N, K,
                          m_tile_group, num_groups, flags, stream);
}

extern "C" int dolomite_b200_gemm_bf16_grouped_k(const void* A, int64_t lda, const void* B, int64_t ldb, float* D,
                                                 int64_t ldd, float alpha, float beta, int64_t M, int64_t N,
                                                 int64_t K_max, const int32_t* group_k_offsets, int num_groups,
                                                 void* stream) {
    DOLO_REQUIRE(group_k_offsets != nullptr && num_groups > 0, "grouped wgrad: missing offsets");
    GroupArgs ga;
    ga.mode = 2;
    ga.group_k_offsets = group_k_offsets;
    ga.num_groups = num_groups;
    ga.d_group_stride = M * ldd;
    // A, B are both MN-major views of [K_max, M] / [K_max, N] row-major activations; D[g] (+)= A_g^T B_g in fp32
    return gemm_impl(A, lda, 1, B, ldb, 1, D, ldd, 1, beta != 0.f ? D : nullptr, ldd, alpha, beta, nullptr, M, N, K_max, 0,
                     stream, ga);
}

// ---------------------------------------------------------------------------------------------------------------------
// FP8 entry points (te.Linear fprop / dgrad / wgrad under fp8_autocast)
// ---------------------------------------------------------------------------------------------------------------------
extern "C" int dolomite_b200_gemm_fp8(const void* A, int64_t lda, int a_fmt, const void* B, int64_t ldb, int b_fmt,
                                      const float* a_scale_inv, const float* b_scale_inv, void* D, int64_t ldd,
                                      int d_is_f32, const void* C, int64_t ldc, float alpha, float beta, const void* bias,
                                      int64_t M, int64_t N, int64_t K, int split_accumulate, void* stream) {
    DOLO_REQUIRE(M >= 0 && N >= 0 && K >= 0, "gemm_fp8: negative dimension");
    DOLO_REQUIRE((a_fmt == 0 || a_fmt == 1) && (b_fmt == 0 || b_fmt == 1), "gemm_fp8: format must be 0 (e4m3) or 1 (e5m2)");
    if (M == 0 || N == 0) return DOLO_OK;
    GemmMaps maps;
    GemmParams p;
    memset(&p, 0, sizeof(p));
    GemmProblemArgs g{A, lda, B, ldb, D, ldd, C, ldc, bias, alpha, beta, M, N, K, a_scale_inv, b_scale_inv};
    int rc = setup_problem(maps, p, 0, g, 1, 0, 0, d_is_f32, GroupArgs(), BN);
    if (rc) return rc;
    p.n_prob = 1;
    p.num_tiles = p.pr[0].num_m * p.pr[0].num_n;
    p.d_is_f32 = d_is_f32;
    p.num_groups = 1;
    return dispatch_fp8(a_fmt, b_fmt, split_accumulate, maps, p, static_cast<cudaStream_t>(stream));
}

extern "C" int dolomite_b200_gemm_fp8_wgrad_multi(int n_problems, const void* const* dYt, const int64_t* ld_dyt,
                                                  const void* const* Xt, const int64_t* ld_xt,
                                                  const float* const* dy_scale_inv, const float* const* x_scale_inv,
                                                  float* const* dW, const int64_t* ld_dw, const int64_t* M,
                                                  const int64_t* N, int64_t K, const float* alpha, const int* accumulate,
                                                  int dy_fmt, int x_fmt, int split_accumulate, void* stream) {
    DOLO_REQUIRE(n_problems >= 1 && n_problems <= MAXP, "gemm_fp8_wgrad_multi: between 1 and %d problems per launch", MAXP);
    DOLO_REQUIRE((dy_fmt == 0 || dy_fmt == 1) && (x_fmt == 0 || x_fmt == 1),
                 "gemm_fp8_wgrad_multi: format must be 0 (e4m3) or 1 (e5m2)");
    GemmMaps maps;
    GemmParams p;
    memset(&p, 0, sizeof(p));
    int tiles = 0;
    for (int q = 0; q < n_problems; ++q) {
        GemmProblemArgs g{dYt[q], ld_dyt[q], Xt[q], ld_xt[q], dW[q], ld_dw[q], accumulate[q] ? dW[q] : nullptr, ld_dw[q],
                          nullptr, alpha[q], 1.f, M[q], N[q], K, dy_scale_inv[q], x_scale_inv[q]};
        int rc = setup_problem(maps, p, q, g, 1, 0, 0, 1, GroupArgs(), BN);
        if (rc) return rc;
        p.pr[q].tile_start = tiles;
        tiles += p.pr[q].num_m * p.pr[q].num_n;
    }
    p.n_prob = n_problems;
    p.num_tiles = tiles;
    p.d_is_f32 = 1;
    p.num_groups = 1;
    return dispatch_fp8(dy_fmt, x_fmt, split_accumulate, maps, p, static_cast<cudaStream_t>(stream));
}
