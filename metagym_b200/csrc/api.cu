// Library-wide entry points of libmgb200: error string, version, device probe.
#include <string.h>

#include "mgb_common.cuh"

static thread_local char g_err[512] = "";

void mgb_set_error(const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

extern "C" const char *mgb_last_error(void) { return g_err; }

extern "C" const char *mgb_version(void) { return "metagym_b200 0.1 (sm_90a)"; }

extern "C" int mgb_device_count(void)
{
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess) {
        mgb_set_error("cudaGetDeviceCount -> %s", cudaGetErrorString(e));
        cudaGetLastError();
        return MGB_ERR_CUDA;
    }
    return n;
}

// ---- peer memory (cudaIpc over NVLink peer mappings), see mgb200.h
extern "C" int mgb_peer_alloc(int device, uint64_t bytes, void **ptr_out)
{
    MGB_REQUIRE(ptr_out && bytes > 0, "bad argument");
    MgbDeviceGuard guard(device);
    MGB_REQUIRE(guard.ok, "cannot select device");
    MgbDev<uint8_t> p;
    MGB_CUDA(p.alloc(bytes));                 // plain cudaMalloc: the only kind cudaIpcGetMemHandle accepts
    MGB_CUDA(cudaMemset(p.get(), 0, bytes));
    MGB_CUDA(cudaDeviceSynchronize());
    *ptr_out = p.release();                   // the caller owns it from here (mgb_peer_free)
    return MGB_OK;
}

extern "C" int mgb_peer_free(int device, void *ptr)
{
    MgbDeviceGuard guard(device);
    MGB_REQUIRE(guard.ok, "cannot select device");
    MGB_CUDA(cudaFree(ptr));
    return MGB_OK;
}

extern "C" int mgb_peer_export(int device, void *ptr, uint8_t handle_out[MGB_PEER_HANDLE_BYTES])
{
    static_assert(sizeof(cudaIpcMemHandle_t) == MGB_PEER_HANDLE_BYTES, "handle size");
    MGB_REQUIRE(ptr && handle_out, "null argument");
    MgbDeviceGuard guard(device);
    MGB_REQUIRE(guard.ok, "cannot select device");
    cudaIpcMemHandle_t hd;
    MGB_CUDA(cudaIpcGetMemHandle(&hd, ptr));
    memcpy(handle_out, &hd, sizeof(hd));
    return MGB_OK;
}

extern "C" int mgb_peer_open(int device, const uint8_t handle[MGB_PEER_HANDLE_BYTES], void **ptr_out)
{
    MGB_REQUIRE(handle && ptr_out, "null argument");
    MgbDeviceGuard guard(device);
    MGB_REQUIRE(guard.ok, "cannot select device");
    cudaIpcMemHandle_t hd;
    memcpy(&hd, handle, sizeof(hd));
    void *p = nullptr;
    MGB_CUDA(cudaIpcOpenMemHandle(&p, hd, cudaIpcMemLazyEnablePeerAccess));
    *ptr_out = p;
    return MGB_OK;
}

extern "C" int mgb_peer_close(int device, void *ptr)
{
    MgbDeviceGuard guard(device);
    MGB_REQUIRE(guard.ok, "cannot select device");
    MGB_CUDA(cudaIpcCloseMemHandle(ptr));
    return MGB_OK;
}
