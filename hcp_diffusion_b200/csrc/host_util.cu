// SPDX-License-Identifier: Apache-2.0
#include "host_util.h"
#include "../../include/hcp_b200.h"
#include <stdio.h>
#include <stdlib.h>
#include <atomic>
#include <mutex>

namespace hcp {

static thread_local char g_err[512] = "ok";

int set_error(int code, const char* msg) {
    snprintf(g_err, sizeof(g_err), "%s", msg);
    return code;
}
int set_cuda_error(cudaError_t e, const char* where) {
    snprintf(g_err, sizeof(g_err), "%s: %s (%s)", where, cudaGetErrorString(e), cudaGetErrorName(e));
    return HCP_ERR_CUDA;
}

int num_sms() {
    static const int n = [] {
        int dev = 0, v = 0;
        if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0)
            return 132;                     // H100 SXM
        return v;
    }();
    return n;
}

static std::atomic<unsigned long long> g_launches{0};
void note_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

bool pdl_enabled() {
    static const bool on = [] {
        // programmatic edges let a kernel's prologue overlap its predecessor's tail inside the captured step graph.
        // HCP_PDL=0 turns them off.
        const char* e = getenv("HCP_PDL");
        return !(e && e[0] == '0');
    }();
    return on;
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
    static PFN_encodeTiled fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
        if (e == cudaSuccess && q == cudaDriverEntryPointSuccess) fn = reinterpret_cast<PFN_encodeTiled>(p);
    });
    return fn;
}

int make_tmap_nd(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                 const uint32_t* box, bool swizzle128) {
    // cuTensorMapEncodeTiled is a driver call and needs a context current on THIS thread; autograd worker threads may
    // not have touched the runtime yet (observed: CUDA_ERROR_INVALID_CONTEXT from a backward thread).  cudaSetDevice on
    // the thread's current device binds its primary context (and, unlike cudaFree(0), is legal during stream capture).
    static thread_local bool ctx_bound = false;
    if (!ctx_bound) {
        int dev = 0;
        cudaError_t e = cudaGetDevice(&dev);
        if (e == cudaSuccess) e = cudaSetDevice(dev);
        if (e != cudaSuccess) return set_cuda_error(e, "cudaSetDevice (context bind)");
        ctx_bound = true;
    }
    PFN_encodeTiled enc = get_encode();
    if (!enc) return set_error(HCP_ERR_NO_DEVICE, "cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
    if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) return set_error(HCP_ERR_INVALID, "tensor map: base not 16-byte aligned");
    cuuint64_t gd[5];
    cuuint64_t gs[4];
    cuuint32_t bx[5];
    cuuint32_t es[5];
    for (int i = 0; i < rank; ++i) {
        gd[i] = dims[i];
        bx[i] = box[i];
        es[i] = 1;
        if (box[i] == 0 || box[i] > 256) return set_error(HCP_ERR_INVALID, "tensor map: box extent out of range");
    }
    for (int i = 0; i + 1 < rank; ++i) {
        gs[i] = strides_bytes[i];
        if (gs[i] % 16 != 0) return set_error(HCP_ERR_INVALID, "tensor map: stride not a multiple of 16 bytes");
    }
    CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(base), gd, gs, bx, es,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        char buf[256];
        snprintf(buf, sizeof(buf), "cuTensorMapEncodeTiled failed (CUresult %d) rank=%d dims=[%llu,%llu,..] box=[%u,%u,..]",
                 (int)r, rank, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0), box[0],
                 rank > 1 ? box[1] : 0);
        return set_error(HCP_ERR_CUDA, buf);
    }
    return HCP_OK;
}

}  // namespace hcp

extern "C" int hcp_version(void) { return 2; }
extern "C" unsigned long long hcp_launch_count(void) { return hcp::g_launches.load(std::memory_order_relaxed); }
extern "C" const char* hcp_last_error_string(void) { return hcp::g_err; }
extern "C" int hcp_device_check(void) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return hcp::set_cuda_error(e, "cudaGetDevice");
    int major = 0, minor = 0;
    e = cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
    if (e != cudaSuccess) return hcp::set_cuda_error(e, "cudaDeviceGetAttribute");
    // the kernels are built for sm_90a only (wgmma): their cubin loads on compute capability 9.0 and nothing else
    if (major != 9 || minor != 0) return hcp::set_error(HCP_ERR_NO_DEVICE, "libhcpb200 needs a compute-capability 9.0 (H100) device");
    return HCP_OK;
}
