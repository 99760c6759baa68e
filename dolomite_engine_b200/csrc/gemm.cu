// bf16 GEMM for sm_90a (H100):  TMA (cp.async.bulk.tensor) -> 128B-swizzled smem ring -> wgmma (m64n128k16 per consumer
// warpgroup, fp32 accumulators in registers) -> epilogue straight from the registers (alpha / bias / beta*C, bf16 | fp32).
//
// Persistent, warp-specialised: warpgroup 0 = producer (one elected thread issues the TMA loads; the whole first warp for
// gather-on-load), warpgroups 1 and 2 = consumers, each owning 64 rows of the 128 x 128 output tile.
// Both operands may be K-major (row-major [rows, K]) or MN-major (stored [K, rows]); the latter is what dgrad / wgrad
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
constexpr int BN = 128;
constexpr int BK = 64;  // 64 bf16 = 128 bytes = one swizzle span
constexpr int STAGES = 6;
constexpr int A_STAGE_BYTES = BM * BK * 2;  // 16 KB
constexpr int B_STAGE_BYTES = BN * BK * 2;  // 16 KB
constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
constexpr int GEMM_THREADS = 384;  // warpgroup 0 producer, 1..2 consumers
constexpr int SMEM_BYTES = 1024 /*align slack*/ + STAGES * STAGE_BYTES + 256 /*barriers*/;
static_assert(SMEM_BYTES <= 232448, "shared memory budget exceeded (227 KB per block on sm_90)");

constexpr int MAXP = 4;  // problems per launch (the four weight gradients of a transformer block share one launch)

struct GemmMaps {
    CUtensorMap a[MAXP], b[MAXP];
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
    //   1 = M-grouped: every 128-row tile of A/D belongs to one group (m_tile_group[m_blk], -1 = unused tile); B's outer
    //       TMA coordinate is offset by group * b_group_rows (fwd / dgrad of the expert linears)
    //   2 = K-grouped: tile index also enumerates the group; the contraction runs over rows
    //       [group_k_offsets[g], group_k_offsets[g+1]) and D/C are offset by g * d_group_stride (expert wgrad)
    int grouped;
    const int* m_tile_group;
    const int* a_row_index;  // gather-on-load: source row of A for every (grouped) row of the problem, or NULL
    const void* gather_a;    // gather-on-load: the ungrouped A [a_rows, K] (row stride gather_lda), read by the producer warp
    int64_t gather_lda;
    int gather_k;
    int b_group_rows;
    const int* group_k_offsets;
    int num_groups;
    int64_t d_group_stride;
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
    if (p.grouped == 3) {
        // split-K: tile index also enumerates the K split; partial products are reduced with fp32 atomics
        const int per = pr.num_m * pr.num_n;
        const int split = t / per;
        tile_coords(t - split * per, pr.num_m, pr.num_n, pr.group_m, ti.m_blk, ti.n_blk);
        const int kb_per = (pr.num_kb + p.num_groups - 1) / p.num_groups;
        ti.kb0 = split * kb_per;
        ti.kb1 = min(pr.num_kb, ti.kb0 + kb_per);
        ti.valid = ti.kb1 > ti.kb0;
    } else if (p.grouped == 2) {
        const int per = pr.num_m * pr.num_n;
        ti.grp = t / per;
        tile_coords(t - ti.grp * per, pr.num_m, pr.num_n, pr.group_m, ti.m_blk, ti.n_blk);
        ti.kb0 = p.group_k_offsets[ti.grp] / BK;
        ti.kb1 = p.group_k_offsets[ti.grp + 1] / BK;
        ti.valid = ti.kb1 > ti.kb0;
    } else {
        tile_coords(t, pr.num_m, pr.num_n, pr.group_m, ti.m_blk, ti.n_blk);
        if (p.grouped == 1) {
            ti.grp = p.m_tile_group[ti.m_blk];
            ti.valid = ti.grp >= 0;
        }
    }
    return ti;
}

template <bool A_MN, bool B_MN>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
    gemm_bf16_kernel(const __grid_constant__ GemmMaps maps, const __grid_constant__ GemmParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_align_1024(smem_raw);
    uint8_t* smem_a = smem;
    uint8_t* smem_b = smem + STAGES * A_STAGE_BYTES;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
    uint64_t* full_bar = bars;            // [STAGES]
    uint64_t* empty_bar = bars + STAGES;  // [STAGES]

    const int wg = threadIdx.x >> 7;
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int num_tiles = p.num_tiles;
    const bool gather = !A_MN && p.a_row_index != nullptr;

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
        mbar_fence_init();
    }
    __syncthreads();

    if (wg == 0) {
        // ================= producer =================
        if (warp != 0) return;
        if (gather) {
            // Gather-on-load (grouped expert GEMM reading the UNGROUPED activations): lane l copies rows 4l .. 4l+3 of the
            // 128-row A tile from their source rows into the 128B-swizzled stage (16-byte chunk c of row r lands at chunk
            // c ^ (r % 8), the layout TMA would have written); lane 0 also loads B through TMA.
            const __nv_bfloat16* A = static_cast<const __nv_bfloat16*>(p.gather_a);
            int stage = 0;
            uint32_t phase = 0;
            for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
                const TileInfo ti = tile_info(t, p);
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
                const TileInfo ti = tile_info(t, p);
                if (!ti.valid) continue;
                const CUtensorMap* tmap_a = &maps.a[ti.q];
                const CUtensorMap* tmap_b = &maps.b[ti.q];
                const uint64_t ha = p.pr[ti.q].hint_a, hb = p.pr[ti.q].hint_b;
                const int m_blk = ti.m_blk, n_blk = ti.n_blk;
                const int b_outer = (p.grouped == 1) ? ti.grp * p.b_group_rows : 0;
                for (int kb = ti.kb0; kb < ti.kb1; ++kb) {
                    mbar_wait(&empty_bar[stage], phase ^ 1, 1);
                    uint8_t* sa = smem_a + stage * A_STAGE_BYTES;
                    uint8_t* sb = smem_b + stage * B_STAGE_BYTES;
                    mbar_expect_tx(&full_bar[stage], STAGE_BYTES);
                    if (!A_MN) {
                        tma_load_2d_hint(sa, tmap_a, &full_bar[stage], kb * BK, m_blk * BM, ha);
                    } else {
#pragma unroll
                        for (int i = 0; i < BM / 64; ++i)
                            tma_load_2d_hint(sa + i * (BK * 128), tmap_a, &full_bar[stage], m_blk * BM + i * 64, kb * BK, ha);
                    }
                    if (!B_MN) {
                        tma_load_2d_hint(sb, tmap_b, &full_bar[stage], kb * BK, b_outer + n_blk * BN, hb);
                    } else {
#pragma unroll
                        for (int i = 0; i < BN / 64; ++i)
                            tma_load_2d_hint(sb + i * (BK * 128), tmap_b, &full_bar[stage], n_blk * BN + i * 64,
                                             b_outer + kb * BK, hb);
                    }
                    if (++stage == STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
        return;
    }

    // ================= consumers: warpgroup cw owns rows [64 cw, 64 cw + 64) of the tile =================
    const int cw = wg - 1;
    const int wr = (warp & 3) * 16 + (lane >> 2);  // accumulator row of this thread inside the warpgroup (and +8)
    const int wc = 2 * (lane & 3);                 // first accumulator column inside each n8 block
    int stage = 0;
    uint32_t phase = 0;
    float acc[BN / 2];
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        const TileInfo ti = tile_info(t, p);
        const Problem& pr = p.pr[ti.q];
        const int64_t row0 = int64_t(ti.m_blk) * BM + cw * 64 + wr;
        const int col0 = ti.n_blk * BN + wc;
        if (!ti.valid) {
            // K-grouped launch (expert weight gradients) and this expert received NO rows: its product is zero.  A launch
            // that OVERWRITES (beta = 0, no C) must still write the tile -- the caller did not clear the buffer.
            if (p.grouped == 2 && p.d_is_f32 && pr.C == nullptr) {
                float* D = static_cast<float*>(pr.D) + int64_t(ti.grp) * p.d_group_stride;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int64_t row = row0 + 8 * h;
                    if (row >= pr.M) continue;
                    for (int j = 0; j < BN / 8; ++j)
                        if (col0 + 8 * j < pr.N)
                            *reinterpret_cast<float2*>(D + row * pr.ldd + col0 + 8 * j) = make_float2(0.f, 0.f);
                }
            }
            continue;
        }
        int prev_stage = -1;
        for (int kb = ti.kb0; kb < ti.kb1; ++kb) {
            mbar_wait(&full_bar[stage], phase, 3);
            wgmma_fence();
            const uint32_t sa = smem_u32(smem_a + stage * A_STAGE_BYTES);
            const uint32_t sb = smem_u32(smem_b + stage * B_STAGE_BYTES);
#pragma unroll
            for (int k = 0; k < BK / 16; ++k) {
                // K-major: +32 B per K=16 step inside the 128 B swizzle span; SBO = 8 rows x 128 B; this warpgroup's
                // 64 rows start 64 x 128 B into the tile.
                // MN-major: +16 K-rows x 128 B per step; LBO = next 64-wide MN chunk (BK rows x 128 B), SBO = 8 K-rows;
                // this warpgroup's 64 rows are the cw-th chunk.
                const uint64_t adesc = A_MN ? gmma_desc(sa + cw * (BK * 128) + k * 2048, BK * 128, 1024, 1)
                                            : gmma_desc(sa + cw * (64 * 128) + k * 32, 16, 1024, 1);
                const uint64_t bdesc = B_MN ? gmma_desc(sb + k * 2048, BK * 128, 1024, 1) : gmma_desc(sb + k * 32, 16, 1024, 1);
                wgmma_ss<BN, A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, adesc, bdesc, (kb != ti.kb0 || k != 0) ? 1u : 0u);
            }
            wgmma_commit();
            wgmma_wait<1>();  // the previous k-block's MMAs retired: its stage may be refilled
            if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);
            prev_stage = stage;
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        reg_fence<BN / 2>(acc);
        if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);

        // ---------------- epilogue: registers -> global ----------------
        const int64_t d_off = (p.grouped == 2) ? int64_t(ti.grp) * p.d_group_stride : 0;
        const float alpha = pr.alpha, beta = pr.beta;
        const __nv_bfloat16* bias = pr.bias;
        const int N = pr.N;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
            const int col = col0 + 8 * j;
            if (col >= N) continue;  // N % 8 == 0: the column pair is either wholly in range or wholly out
            float b0 = 0.f, b1 = 0.f;
            if (bias != nullptr) {
                const uint32_t bv = *reinterpret_cast<const uint32_t*>(bias + col);
                b0 = bf16_lo(bv);
                b1 = bf16_hi(bv);
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int64_t row = row0 + 8 * h;
                if (row >= pr.M) continue;
                float v0 = (acc[4 * j + 2 * h] + b0) * alpha;
                float v1 = (acc[4 * j + 2 * h + 1] + b1) * alpha;
                if (p.d_is_f32) {
                    float* d = static_cast<float*>(pr.D) + d_off + row * pr.ldd + col;
                    if (p.grouped == 3) {  // split-K partial: D += v
                        asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(d), "f"(v0), "f"(v1) : "memory");
                        continue;
                    }
                    if (pr.C) {
                        const float2 c2 = *reinterpret_cast<const float2*>(static_cast<const float*>(pr.C) + d_off + row * pr.ldc + col);
                        v0 += beta * c2.x;
                        v1 += beta * c2.y;
                    }
                    *reinterpret_cast<float2*>(d) = make_float2(v0, v1);
                } else {
                    __nv_bfloat16* d = static_cast<__nv_bfloat16*>(pr.D) + d_off + row * pr.ldd + col;
                    if (pr.C) {
                        const uint32_t cv =
                            *reinterpret_cast<const uint32_t*>(static_cast<const __nv_bfloat16*>(pr.C) + d_off + row * pr.ldc + col);
                        v0 += beta * bf16_lo(cv);
                        v1 += beta * bf16_hi(cv);
                    }
                    *reinterpret_cast<uint32_t*>(d) = pack_bf16(v0, v1);
                }
            }
        }
    }
}

template <bool A_MN, bool B_MN>
int launch_gemm(const GemmMaps& maps, const GemmParams& p, cudaStream_t st) {
    auto kern = gemm_bf16_kernel<A_MN, B_MN>;
    static bool attr_set = false;  // per instantiation
    if (!attr_set) {
        DOLO_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
        attr_set = true;
    }
    // static persistent schedule: worker w takes tiles w, w + W, ... on `SMs - gemm_sm_margin` SMs
    int sms = dolo_num_sms() - dolo_option_gemm_sm_margin();
    if (sms < 1) sms = 1;
    const int grid = p.num_tiles < sms ? p.num_tiles : sms;
    kern<<<grid, GEMM_THREADS, SMEM_BYTES, st>>>(maps, p);
    DOLO_LAUNCH_OK("gemm_bf16");
    return DOLO_OK;
}

}  // namespace

struct GroupArgs {
    int mode = 0;
    const int* a_row_index = nullptr;  // mode 1 only: gather the rows of A on load (A is the ungrouped matrix of a_rows rows)
    int64_t a_rows = 0;
    const int* m_tile_group = nullptr;
    int64_t b_group_rows = 0;
    const int* group_k_offsets = nullptr;
    int num_groups = 1;
    int64_t d_group_stride = 0;
    int64_t b_total_outer = 0;  // rows of B's outer TMA dimension over all groups
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
};

// Fills maps.{a,b}[q] and p.pr[q] for one problem.  All problems of a launch share the operand layouts and the output type.
static int setup_problem(GemmMaps& maps, GemmParams& p, int q, const GemmProblemArgs& g, int a_mn_major, int b_mn_major,
                         int d_is_f32, const GroupArgs& ga) {
    const int64_t M = g.M, N = g.N, K = g.K;
    DOLO_REQUIRE(K > 0, "gemm: K must be > 0");
    DOLO_REQUIRE(K % 8 == 0 && N % 8 == 0, "gemm: K=%lld and N=%lld must be multiples of 8", (long long)K, (long long)N);
    DOLO_REQUIRE(g.lda % 8 == 0 && g.ldb % 8 == 0 && g.ldd % (d_is_f32 ? 4 : 8) == 0,
                 "gemm: leading dimensions must keep 16-byte alignment");
    DOLO_REQUIRE(!a_mn_major || M % 8 == 0, "gemm: MN-major A requires M %% 8 == 0");
    DOLO_REQUIRE(g.C == nullptr || g.ldc % (d_is_f32 ? 4 : 8) == 0, "gemm: ldc alignment");
    DOLO_REQUIRE(M < (1ll << 31) && N < (1ll << 31) && K < (1ll << 31), "gemm: dimension too large");
    // K-major: dims {K, rows}, box {64, tile rows}.  MN-major: dims {rows, K}, box {64, 64}.
    uint64_t dims[2], strides[2];
    uint32_t box[2];
    int rc;
    if (ga.a_row_index != nullptr) {
        // gather-on-load: the producer warp reads A's rows itself (no tensor map)
        DOLO_REQUIRE(!a_mn_major, "gemm: gather-on-load needs a K-major A");
        DOLO_REQUIRE((reinterpret_cast<uintptr_t>(g.A) & 15) == 0, "gemm: gather-on-load needs a 16-byte aligned A");
        p.gather_a = g.A;
        p.gather_lda = g.lda;
        p.gather_k = int(K);
    } else {
        if (!a_mn_major) {
            dims[0] = uint64_t(K); dims[1] = uint64_t(M); strides[0] = 2; strides[1] = uint64_t(g.lda) * 2;
            box[0] = BK; box[1] = BM;
        } else {
            dims[0] = uint64_t(M); dims[1] = uint64_t(K); strides[0] = 2; strides[1] = uint64_t(g.lda) * 2;
            box[0] = 64; box[1] = BK;
        }
        rc = dolo_make_tmap(&maps.a[q], g.A, 2, 2, dims, strides, box, DOLO_SW_128);
        if (rc) return rc;
    }
    strides[0] = 2;
    if (!b_mn_major) {
        dims[0] = uint64_t(K); dims[1] = uint64_t(ga.mode == 1 ? ga.b_total_outer : N); strides[1] = uint64_t(g.ldb) * 2;
        box[0] = BK; box[1] = BN;
    } else {
        dims[0] = uint64_t(N); dims[1] = uint64_t(ga.mode == 1 ? ga.b_total_outer : K); strides[1] = uint64_t(g.ldb) * 2;
        box[0] = 64; box[1] = BK;
    }
    rc = dolo_make_tmap(&maps.b[q], g.B, 2, 2, dims, strides, box, DOLO_SW_128);
    if (rc) return rc;
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
    if (dolo_option_gemm_l2_hints() && ga.mode == 0 && K >= 4096 && (M + N) * K * 2 > (24ll << 20)) {
        // long contraction, operands larger than what the L2 keeps anyway: stream the bigger one, keep the smaller one
        const bool a_smaller = M <= N;
        pr.hint_a = a_smaller ? TMA_HINT_EVICT_LAST : TMA_HINT_EVICT_FIRST;
        pr.hint_b = a_smaller ? TMA_HINT_EVICT_FIRST : TMA_HINT_EVICT_LAST;
    }
    pr.num_m = int((M + BM - 1) / BM);
    pr.num_n = int((N + BN - 1) / BN);
    pr.num_kb = int((K + BK - 1) / BK);
    {
        // A panel of group_m x 128 rows x K bf16 should fit comfortably in the 50 MB L2 next to the streaming B tiles
        const int64_t panel_bytes = int64_t(BM) * K * 2;
        int64_t gm = (12ll << 20) / (panel_bytes > 0 ? panel_bytes : 1);
        if (gm < 4) gm = 4;
        if (gm > 64) gm = 64;
        pr.group_m = int(gm);
    }
    return DOLO_OK;
}

template <typename... Ts>
static int dispatch_layout(int a_mn_major, int b_mn_major, Ts&&... args) {
    if (!a_mn_major && !b_mn_major) return launch_gemm<false, false>(args...);
    if (!a_mn_major && b_mn_major) return launch_gemm<false, true>(args...);
    if (a_mn_major && !b_mn_major) return launch_gemm<true, false>(args...);
    return launch_gemm<true, true>(args...);
}

static int gemm_impl(const void* A, int64_t lda, int a_mn_major, const void* B, int64_t ldb, int b_mn_major, void* D,
                     int64_t ldd, int d_is_f32, const void* C, int64_t ldc, float alpha, float beta, const void* bias,
                     int64_t M, int64_t N, int64_t K, int flags, void* stream, const GroupArgs& ga) {
    DOLO_REQUIRE(M >= 0 && N >= 0 && K >= 0, "gemm: negative dimension");
    if (M == 0 || N == 0) return DOLO_OK;
    const bool tma_store = (flags & DOLO_GEMM_FLAG_TMA_STORE) != 0;
    DOLO_REQUIRE(!tma_store || (!d_is_f32 && C == nullptr), "gemm: TMA-store epilogue needs bf16 D and no C");
    GemmMaps maps;
    GemmParams p;
    memset(&p, 0, sizeof(p));
    GemmProblemArgs g{A, lda, B, ldb, D, ldd, C, ldc, bias, alpha, beta, M, N, K};
    int rc = setup_problem(maps, p, 0, g, a_mn_major, b_mn_major, d_is_f32, ga);
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
    p.d_group_stride = ga.d_group_stride;
    return dispatch_layout(a_mn_major, b_mn_major, maps, p, static_cast<cudaStream_t>(stream));
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
    GemmMaps maps;
    GemmParams p;
    memset(&p, 0, sizeof(p));
    int tiles = 0;
    for (int q = 0; q < n_problems; ++q) {
        DOLO_REQUIRE(M[q] > 0 && N[q] > 0, "wgrad_multi: empty problem %d", q);
        GemmProblemArgs g{dY[q], ld_dy[q], X[q], ld_x[q], dW[q], ld_dw[q], accumulate[q] ? dW[q] : nullptr, ld_dw[q], nullptr,
                          alpha[q], 1.f, M[q], N[q], K};
        int rc = setup_problem(maps, p, q, g, 1, 1, 1, GroupArgs());
        if (rc) return rc;
        p.pr[q].tile_start = tiles;
        tiles += p.pr[q].num_m * p.pr[q].num_n;
    }
    p.n_prob = n_problems;
    p.num_tiles = tiles;
    p.d_is_f32 = 1;
    p.grouped = 0;
    p.num_groups = 1;
    return launch_gemm<true, true>(maps, p, static_cast<cudaStream_t>(stream));
}

extern "C" int dolomite_b200_gemm_bf16(const void* A, int64_t lda, int a_mn_major, const void* B, int64_t ldb,
                                       int b_mn_major, void* D, int64_t ldd, int d_is_f32, const void* C, int64_t ldc,
                                       float alpha, float beta, const void* bias, int64_t M, int64_t N, int64_t K,
                                       int flags, void* stream) {
    if (flags & DOLO_GEMM_FLAG_SPLITK_ACCUMULATE) {
        // D(fp32) += alpha * A B^T with the contraction split over several CTAs (fp32 vector atomics): removes the
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

extern "C" int dolomite_b200_gemm_bf16_grouped_m(const void* A, int64_t lda, const void* B, int64_t ldb, int b_mn_major,
                                                 void* D, int64_t ldd, float alpha, int64_t M_max, int64_t N, int64_t K,
                                                 const int32_t* m_tile_group, int num_groups, int flags, void* stream) {
    DOLO_REQUIRE(M_max % BM == 0, "grouped gemm: M_max=%lld must be a multiple of %d (padded expert segments)",
                 (long long)M_max, BM);
    DOLO_REQUIRE(!b_mn_major || K % BK == 0, "grouped gemm: MN-major B needs K %% %d == 0", BK);
    DOLO_REQUIRE(m_tile_group != nullptr && num_groups > 0, "grouped gemm: missing group table");
    GroupArgs ga;
    ga.mode = 1;
    ga.m_tile_group = m_tile_group;
    ga.num_groups = num_groups;
    ga.b_group_rows = b_mn_major ? K : N;
    ga.b_total_outer = ga.b_group_rows * num_groups;
    return gemm_impl(A, lda, 0, B, ldb, b_mn_major, D, ldd, 0, nullptr, 0, alpha, 0.f, nullptr, M_max, N, K, flags, stream,
                     ga);
}

// Same, with the ScatterMoE gather fused into the operand load: A is the UNGROUPED activation matrix [a_rows, K] and
// a_row_index[r] names the source row of grouped row r (padding rows may name any valid row: their products are never read)
extern "C" int dolomite_b200_gemm_bf16_grouped_m_gather(const void* A, int64_t lda, int64_t a_rows,
                                                        const int32_t* a_row_index, const void* B, int64_t ldb, void* D,
                                                        int64_t ldd, float alpha, int64_t M_max, int64_t N, int64_t K,
                                                        const int32_t* m_tile_group, int num_groups, int flags,
                                                        void* stream) {
    DOLO_REQUIRE(M_max % BM == 0, "grouped gemm: M_max=%lld must be a multiple of %d (padded expert segments)",
                 (long long)M_max, BM);
    DOLO_REQUIRE(m_tile_group != nullptr && num_groups > 0 && a_row_index != nullptr && a_rows > 0,
                 "grouped gemm (gather): missing group table / row index");
    DOLO_REQUIRE((reinterpret_cast<uintptr_t>(a_row_index) & 15) == 0, "grouped gemm (gather): row index must be 16-byte aligned");
    GroupArgs ga;
    ga.mode = 1;
    ga.a_row_index = a_row_index;
    ga.a_rows = a_rows;
    ga.m_tile_group = m_tile_group;
    ga.num_groups = num_groups;
    ga.b_group_rows = N;
    ga.b_total_outer = N * num_groups;
    return gemm_impl(A, lda, 0, B, ldb, 0, D, ldd, 0, nullptr, 0, alpha, 0.f, nullptr, M_max, N, K, flags, stream, ga);
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
