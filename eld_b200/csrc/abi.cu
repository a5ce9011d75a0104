// abi.cu - context management and error channel of the C ABI (include/eld_b200.h).
#include "common.cuh"
#include "unet_prims.h"
#include <cstring>
#include <new>

namespace eld {
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
}  // namespace eld

extern "C" {

int eld_abi_version(void) { return ELD_ABI_VERSION; }

const char* eld_last_error(void) { return eld::g_err; }

int eld_ctx_create(int device, eld_ctx** out)
{
    ELD_REQUIRE(out != nullptr, "eld_ctx_create: out is NULL");
    *out = nullptr;
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count <= 0) {
        eld::set_error("eld_ctx_create: no CUDA device (%s); this library has no CPU fallback",
                       e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
        return ELD_E_CUDA;
    }
    ELD_REQUIRE(device >= 0 && device < count, "eld_ctx_create: device %d out of range [0,%d)", device, count);
    ELD_CHECK_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    ELD_CHECK_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) {
        eld::set_error("eld_ctx_create: device %d is sm_%d%d; this library is built for sm_90a only",
                       device, prop.major, prop.minor);
        return ELD_E_UNSUPPORTED;
    }
    eld_ctx* ctx = new (std::nothrow) eld_ctx();
    ELD_REQUIRE(ctx != nullptr, "eld_ctx_create: out of host memory");
    ctx->device = device;
    ctx->num_sms = prop.multiProcessorCount;
    ctx->smem_optin = (int)prop.sharedMemPerBlockOptin;
    ctx->launches.store(0);
    // TMA descriptors are encoded by the driver; fetch the entry point through the runtime so the
    // library carries no link-time dependency on libcuda.so (absent on the build box).
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || fn == nullptr) {
        eld::set_error("eld_ctx_create: cuTensorMapEncodeTiled unavailable (%s)",
                       e == cudaSuccess ? "query failed" : cudaGetErrorString(e));
        delete ctx;
        return ELD_E_CUDA;
    }
    ctx->encode_tiled = (eld::PFN_encodeTiled)fn;
    { int rc = eld::init_gemm_kernels(ctx); if (rc != ELD_OK) { delete ctx; return rc; } }
    *out = ctx;
    return ELD_OK;
}

void eld_ctx_destroy(eld_ctx* ctx) { delete ctx; }

int64_t eld_launch_count(const eld_ctx* ctx) { return ctx ? ctx->launches.load() : 0; }

}  // extern "C"
