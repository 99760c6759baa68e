// C-ABI plumbing: error state, device queries, TMA descriptor encode.
#include <cudaTypedefs.h>
#include <stdarg.h>
#include <string.h>

#include "common.cuh"
#include "../../include/dolomite_b200.h"

static thread_local char g_err[1024] = {0};

int dolo_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return DOLO_ERR_INVALID;
}

int dolo_check_cuda(cudaError_t e, const char* what) {
    snprintf(g_err, sizeof(g_err), "CUDA error %d (%s) at %s", int(e), cudaGetErrorString(e), what);
    return DOLO_ERR_CUDA;
}

extern "C" const char* dolomite_b200_last_error() { return g_err; }

extern "C" int dolomite_b200_abi_version() { return DOLOMITE_B200_ABI_VERSION; }

// gemm_cta_pair, attn_fwd_split, attn_bwd_variant, attn_bwd_ablate, gemm_dynamic and gemm_f32_tma_epilogue select kernel
// variants of other GPU generations: sm_90 has one kernel for each of these jobs, so their values are only stored and
// reported back (callers written for the ABI keep working).
static int g_gemm_cta_pair = 1;
static int g_gemm_sm_margin = 0;
int dolo_option_gemm_sm_margin() { return g_gemm_sm_margin; }
static int g_attn_fwd_split = 1;
static int g_attn_bwd_variant = 2;
static int g_attn_head_fastest = 8;
int dolo_option_attn_head_fastest() { return g_attn_head_fastest; }
static int g_attn_bwd_ablate = 0;
static int g_gemm_l2_hints = 1;
int dolo_option_gemm_l2_hints() { return g_gemm_l2_hints; }
static int g_gemm_dynamic = 1;
static int g_gemm_f32_tma_epilogue = 0;

extern "C" int dolomite_b200_set_option(const char* key, int value) {
    if (key != nullptr && strcmp(key, "gemm_sm_margin") == 0) {
        DOLO_REQUIRE(value >= 0 && value <= 64, "gemm_sm_margin must be in [0, 64]");
        g_gemm_sm_margin = value;
        return DOLO_OK;
    }
    if (key != nullptr && strcmp(key, "attn_fwd_split") == 0) {
        g_attn_fwd_split = value;
        return DOLO_OK;
    }
    if (key != nullptr && strcmp(key, "attn_bwd_variant") == 0) {
        DOLO_REQUIRE(value >= 0 && value <= 2, "attn_bwd_variant must be 0, 1 or 2");
        g_attn_bwd_variant = value;
        return DOLO_OK;
    }
    if (key != nullptr && strcmp(key, "attn_head_fastest") == 0) {
        DOLO_REQUIRE(value >= 0 && value <= 1024, "attn_head_fastest must be in [0, 1024]");
        g_attn_head_fastest = value;
        return DOLO_OK;
    }
    if (key != nullptr && strcmp(key, "attn_bwd_ablate") == 0) {
        g_attn_bwd_ablate = value;
        return DOLO_OK;
    }
    if (key != nullptr && strcmp(key, "gemm_l2_hints") == 0) {
        g_gemm_l2_hints = value != 0;
        return DOLO_OK;
    }
    if (key != nullptr && strcmp(key, "gemm_f32_tma_epilogue") == 0) {
        g_gemm_f32_tma_epilogue = value != 0;
        return DOLO_OK;
    }
    if (key != nullptr && strcmp(key, "gemm_dynamic") == 0) {
        g_gemm_dynamic = value != 0;
        return DOLO_OK;
    }
    if (key != nullptr && strcmp(key, "gemm_cta_pair") == 0) {
        g_gemm_cta_pair = value != 0;
        return DOLO_OK;
    }
    return dolo_set_error("unknown option '%s'", key ? key : "(null)");
}

extern "C" int dolomite_b200_get_option(const char* key, int* value) {
    DOLO_REQUIRE(key != nullptr && value != nullptr, "get_option: null argument");
    if (strcmp(key, "gemm_sm_margin") == 0) *value = g_gemm_sm_margin;
    else if (strcmp(key, "attn_fwd_split") == 0) *value = g_attn_fwd_split;
    else if (strcmp(key, "attn_bwd_variant") == 0) *value = g_attn_bwd_variant;
    else if (strcmp(key, "attn_bwd_ablate") == 0) *value = g_attn_bwd_ablate;
    else if (strcmp(key, "attn_head_fastest") == 0) *value = g_attn_head_fastest;
    else if (strcmp(key, "gemm_l2_hints") == 0) *value = g_gemm_l2_hints;
    else if (strcmp(key, "gemm_f32_tma_epilogue") == 0) *value = g_gemm_f32_tma_epilogue;
    else if (strcmp(key, "gemm_dynamic") == 0) *value = g_gemm_dynamic;
    else if (strcmp(key, "gemm_cta_pair") == 0) *value = g_gemm_cta_pair;
    else return dolo_set_error("unknown option '%s'", key);
    return DOLO_OK;
}

int dolo_num_sms() {
    static int cached[64] = {0};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
    if (cached[dev] == 0) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
        cached[dev] = n;
    }
    return cached[dev];
}

extern "C" int dolomite_b200_device_info(int* sm_count, int* cc_major, int* cc_minor) {
    int dev = 0;
    DOLO_CUDA_OK(cudaGetDevice(&dev));
    if (sm_count) DOLO_CUDA_OK(cudaDeviceGetAttribute(sm_count, cudaDevAttrMultiProcessorCount, dev));
    if (cc_major) DOLO_CUDA_OK(cudaDeviceGetAttribute(cc_major, cudaDevAttrComputeCapabilityMajor, dev));
    if (cc_minor) DOLO_CUDA_OK(cudaDeviceGetAttribute(cc_minor, cudaDevAttrComputeCapabilityMinor, dev));
    return DOLO_OK;
}

static PFN_cuTensorMapEncodeTiled_v12000 get_encode_fn() {
    static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
    if (fn) return fn;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || p == nullptr) return nullptr;
    fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
    return fn;
}

int dolo_make_tmap(CUtensorMap* out, const void* base, int elem_bytes, int rank, const uint64_t* dims,
                   const uint64_t* strides_bytes, const uint32_t* box, DoloSwizzle sw) {
    // cuTensorMapEncodeTiled is a DRIVER call: it needs a current context on the calling thread.  The autograd
    // backward thread has only a runtime-API device set, so bind the primary context once per thread.
    static thread_local bool ctx_bound = false;
    if (!ctx_bound) {
        DOLO_CUDA_OK(cudaFree(nullptr));
        ctx_bound = true;
    }
    auto fn = get_encode_fn();
    DOLO_REQUIRE(fn != nullptr, "cuTensorMapEncodeTiled driver entry point unavailable (no CUDA driver?)");
    DOLO_REQUIRE(rank >= 1 && rank <= 5, "tensor map rank %d out of range", rank);
    DOLO_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0, "tensor map base %p not 16-byte aligned", base);
    CUtensorMapDataType dt;
    switch (elem_bytes) {
        case 2: dt = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16; break;
        case 4: dt = CU_TENSOR_MAP_DATA_TYPE_FLOAT32; break;
        default: return dolo_set_error("unsupported TMA element size %d", elem_bytes);
    }
    cuuint64_t gdim[5];
    cuuint64_t gstr[5];
    cuuint32_t bx[5];
    cuuint32_t es[5];
    for (int i = 0; i < rank; ++i) {
        gdim[i] = dims[i];
        bx[i] = box[i];
        es[i] = 1;
        if (i >= 1) {
            gstr[i - 1] = strides_bytes[i];
            DOLO_REQUIRE((strides_bytes[i] & 15) == 0, "TMA stride %llu (dim %d) not a multiple of 16 bytes",
                         (unsigned long long)strides_bytes[i], i);
        }
    }
    CUtensorMapSwizzle s = CU_TENSOR_MAP_SWIZZLE_NONE;
    if (sw == DOLO_SW_32) s = CU_TENSOR_MAP_SWIZZLE_32B;
    if (sw == DOLO_SW_64) s = CU_TENSOR_MAP_SWIZZLE_64B;
    if (sw == DOLO_SW_128) s = CU_TENSOR_MAP_SWIZZLE_128B;
    CUresult r = fn(out, dt, rank, const_cast<void*>(base), gdim, gstr, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE, s,
                    CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        return dolo_set_error(
            "cuTensorMapEncodeTiled failed (%d): rank %d dims [%llu,%llu,%llu] stride1 %llu box [%u,%u,%u] sw %d", int(r),
            rank, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
            (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)(rank > 1 ? strides_bytes[1] : 0), box[0],
            rank > 1 ? box[1] : 0, rank > 2 ? box[2] : 0, int(sw));
    }
    return DOLO_OK;
}
