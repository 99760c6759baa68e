// Shared device/host helpers for the dolomite-b200 C-ABI library (sm_90a, H100).
//
// Everything here is hand-written inline PTX for Hopper: mbarrier, TMA (cp.async.bulk.tensor), wgmma descriptors and
// fences (the MMA wrappers themselves are in wgmma.cuh) and a few vector load/store helpers.  No CUTLASS / CuTe types
// are used.
#pragma once

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

// ------------------------------------------------------------------------------------------
// host-side error plumbing (see api.cu)
// ------------------------------------------------------------------------------------------
extern "C" const char* dolomite_b200_last_error();
int dolo_set_error(const char* fmt, ...);
int dolo_check_cuda(cudaError_t e, const char* what);

#define DOLO_CUDA_OK(expr)                                             \
    do {                                                               \
        cudaError_t _e = (expr);                                       \
        if (_e != cudaSuccess) return dolo_check_cuda(_e, #expr);      \
    } while (0)

#define DOLO_REQUIRE(cond, ...)                                        \
    do {                                                               \
        if (!(cond)) return dolo_set_error(__VA_ARGS__);               \
    } while (0)

#define DOLO_LAUNCH_OK(name)                                           \
    do {                                                               \
        cudaError_t _e = cudaGetLastError();                           \
        if (_e != cudaSuccess) return dolo_check_cuda(_e, name);       \
    } while (0)

int dolo_num_sms();
// SMs left free by the persistent GEMM grids.  A persistent grid sized to ALL SMs runs up to 2x longer when a
// communication kernel (NCCL all-gather / reduce-scatter, a few CTAs) occupies some SMs: the GEMM CTAs that do not fit
// only start when a whole persistent CTA retires.  The sharded data-parallel runtime sets this to NCCL's CTA budget.
int dolo_option_gemm_sm_margin();
// attention CTA order (attention_common.cuh: attn_cta_order): heads per chunk (default 8; heads fastest inside a chunk, the
// longest tiles of a document first, so that the last wave holds short tiles only); 0 = tiles fastest
int dolo_option_attn_head_fastest();
int dolo_option_gemm_l2_hints();  // 1 (default) = evict-first / evict-last operand loads for long-contraction GEMMs

// TMA descriptor encode through the driver entry point (no link-time libcuda dependency).
// rank-2 / rank-3 bf16/f32 tiled maps.  dims/strides innermost first; strides in BYTES for dims >= 1.
enum DoloSwizzle { DOLO_SW_NONE = 0, DOLO_SW_32 = 1, DOLO_SW_64 = 2, DOLO_SW_128 = 3 };
int dolo_make_tmap(CUtensorMap* out, const void* base, int elem_bytes, int rank, const uint64_t* dims,
                   const uint64_t* strides_bytes, const uint32_t* box, DoloSwizzle sw);

// ------------------------------------------------------------------------------------------
// device helpers
// ------------------------------------------------------------------------------------------
#ifdef __CUDACC__

namespace dolo {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// 1024-byte aligned start of the dynamic shared memory window.  Pointer arithmetic on the `extern __shared__` symbol
// itself (not a round trip through uintptr_t) keeps the shared address space visible to the compiler, so every access
// through the result compiles to LDS/STS instead of generic LD/ST.
__device__ __forceinline__ uint8_t* smem_align_1024(uint8_t* smem_raw) {
    return smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
}

__device__ __forceinline__ bool elect_one() {
    uint32_t pred = 0;
    asm volatile(
        "{\n\t"
        ".reg .pred P1;\n\t"
        "elect.sync _|P1, 0xffffffff;\n\t"
        "selp.u32 %0, 1, 0, P1;\n\t"
        "}\n"
        : "=r"(pred));
    return pred != 0;
}

// ---------------- mbarrier ----------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}

// Watchdog: a pipeline bug must surface as a trap (reported by the host as a CUDA error), never as a hung GPU.  ~4 s at
// 2 GHz.  No printf here: a function call inside a wgmma pipeline makes ptxas serialise every wgmma of the kernel.
#ifndef DOLO_WATCHDOG_CYCLES
#define DOLO_WATCHDOG_CYCLES (8000000000LL)
#endif
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, int tag = 0) {
    (void)tag;  // identifies the waiting role at the call site
    if (mbar_try_wait(bar, parity)) return;
    long long t0 = clock64();
    while (!mbar_try_wait(bar, parity)) {
        if (clock64() - t0 > DOLO_WATCHDOG_CYCLES) __trap();
    }
}

// ---------------- proxies / fences ----------------
__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ---------------- TMA ----------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
// L2 eviction-priority hints for TMA loads (the fixed policy encodings of the sm_90+ `createpolicy` instruction).  A GEMM
// whose contraction is long streams one operand once per wave of tiles and re-uses the other in every wave: the streamed
// operand is loaded evict-first, the re-used one evict-last, so the re-used panels survive in the 50 MB L2.
constexpr uint64_t TMA_HINT_NORMAL = 0x1000000000000000ull;
constexpr uint64_t TMA_HINT_EVICT_FIRST = 0x12F0000000000000ull;
constexpr uint64_t TMA_HINT_EVICT_LAST = 0x14F0000000000000ull;
__device__ __forceinline__ void tma_load_2d_hint(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                                 uint64_t hint) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4}], [%2], %5;"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "l"(hint)
        : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* smem_src, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                     reinterpret_cast<uint64_t>(m)),
                 "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
                 : "memory");
}
// rank-2 fp32 tile reduce-add (L2 performs the add; element type lives in the tensor map)
__device__ __forceinline__ void tma_reduce_add_2d(const CUtensorMap* m, const void* smem_src, int c0, int c1) {
    asm volatile("cp.reduce.async.bulk.tensor.2d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                     reinterpret_cast<uint64_t>(m)),
                 "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
                 : "memory");
}
// rank-3 tile store / fp32 reduce-add (the element type and the add live in the tensor map / the instruction): the third
// coordinate selects the group of a grouped weight-gradient GEMM (0 for dense problems)
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* m, const void* smem_src, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(
                     reinterpret_cast<uint64_t>(m)),
                 "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2)
                 : "memory");
}
__device__ __forceinline__ void tma_reduce_add_3d(const CUtensorMap* m, const void* smem_src, int c0, int c1, int c2) {
    asm volatile("cp.reduce.async.bulk.tensor.3d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(
                     reinterpret_cast<uint64_t>(m)),
                 "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2)
                 : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
    asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait_all() {
    asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}
// Bulk (TMA engine) fp32 reduce-add of a contiguous shared-memory slab into global memory: one instruction replaces
// bytes/16 per-thread red.global.add.v4.f32 and is applied by the L2 in full lines.  16-byte aligned, size % 16 == 0.
// Belongs to the thread's bulk async-group (tma_store_commit / tma_store_wait_*).
__device__ __forceinline__ void bulk_reduce_add_f32(float* gdst, uint32_t smem_src, uint32_t bytes) {
    asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.f32 [%0], [%1], %2;" ::"l"(gdst),
                 "r"(smem_src), "r"(bytes)
                 : "memory");
}


// ---------------- thread-block clusters ----------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// ---------------- wgmma (sm_90a warpgroup MMA) ----------------
// Shared-memory matrix descriptor of sm_90 wgmma.  layout_type: 0 none, 1 SW128, 2 SW64, 3 SW32.  K-major swizzled
// operands: SBO = byte stride between 8-row groups (LBO unused); MN-major: LBO = byte stride between MN swizzle atoms,
// SBO = byte stride between 8-row groups of the contraction.
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes, uint32_t layout_type) {
    uint64_t d = 0;
    d |= uint64_t((saddr & 0x3FFFFu) >> 4);
    d |= uint64_t((lbo_bytes >> 4) & 0x3FFFu) << 16;
    d |= uint64_t((sbo_bytes >> 4) & 0x3FFFu) << 32;
    d |= uint64_t(layout_type & 3u) << 62;
    return d;
}
// registers of the accumulators / register A operands are ready for (or were written by) wgmma
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
    asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// Compile-time only: ties accumulator registers to the asm stream, so that no read of them is scheduled above a
// wgmma_wait (the asm of the MMA and of the wait do not name them together).
template <int N>
__device__ __forceinline__ void reg_fence(float* d) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}


// ---------------- small numeric helpers ----------------
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
    __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float bf16_lo(uint32_t v) { return __uint_as_float(v << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t v) { return __uint_as_float(v & 0xFFFF0000u); }
__device__ __forceinline__ float bf16_round(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }
// The bf16 A fragment (m64k16, register operand of wgmma) of contraction step kk from an fp32 accumulator whose columns
// are that contraction: n8 blocks 2kk and 2kk + 1 hold exactly the A elements this thread owns.
__device__ __forceinline__ void acc_to_a_frag(const float* d, int kk, uint32_t (&a)[4]) {
    a[0] = pack_bf16(d[8 * kk + 0], d[8 * kk + 1]);
    a[1] = pack_bf16(d[8 * kk + 2], d[8 * kk + 3]);
    a[2] = pack_bf16(d[8 * kk + 4], d[8 * kk + 5]);
    a[3] = pack_bf16(d[8 * kk + 6], d[8 * kk + 7]);
}

// 2^x on the MUFU pipe in ONE instruction (exp2f() adds range fix-ups we do not need: inputs are <= 0 or -inf)
// ---------------- dropout masks (counter-based: the same mask is regenerated in backward and in recomputed blocks) -----------
// keep <=> hash >= threshold with threshold = round(p * 2^32): P(keep) = 1 - p.  `lowbias32` is the 2-multiply integer
// finaliser (xorshift-multiply chain); the generator is this library's own -- torch's Philox stream cannot be reproduced
// by any independent kernel, the distribution (independent Bernoulli(1 - p) masks scaled by 1 / (1 - p)) is what is kept.
// oracle/dolomite_oracle.py restates both functions in numpy (DropoutOracle), bit for bit.
__device__ __forceinline__ uint32_t lowbias32(uint32_t x) {
    x ^= x >> 16;
    x *= 0x21f0aaadu;
    x ^= x >> 15;
    x *= 0x735a2d97u;
    x ^= x >> 15;
    return x;
}
// element e of a flat activation tensor (site keys key0 / key1 from the host: seed and call site)
__device__ __forceinline__ uint32_t dropout_hash_flat(uint64_t e, uint32_t key0, uint32_t key1) {
    return lowbias32(lowbias32(uint32_t(e) ^ key0) + uint32_t(e >> 32) + key1);
}
// attention probability of (query token q, key token k) -- global token rows of the packed stream -- for one head;
// head_key = dropout_head_key(head, key0, key1) is hoisted out of the loops
__device__ __forceinline__ uint32_t dropout_head_key(uint32_t head, uint32_t key0, uint32_t key1) {
    return lowbias32(head * 0xC2B2AE3Du + key0) ^ key1;
}
__device__ __forceinline__ uint32_t dropout_hash_qk(uint32_t q, uint32_t k, uint32_t head_key) {
    return lowbias32((q * 0x9E3779B1u) ^ (k * 0x85EBCA77u) ^ head_key);
}

__device__ __forceinline__ float fast_exp2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

}  // namespace dolo
#endif  // __CUDACC__
