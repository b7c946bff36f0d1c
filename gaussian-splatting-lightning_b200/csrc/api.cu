// Library-wide state of libb200gs.so: the error text, the launch count, the version and the IPC helpers.  Every other entry point of
// include/b200gs.h is defined in the .cu file of its kernels.
#include <stdarg.h>
#include <string.h>

#include <atomic>

#include "common.cuh"

namespace b200gs {

static thread_local char g_error[512] = "";

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_error, sizeof(g_error), fmt, ap);
    va_end(ap);
}

static std::atomic<unsigned long long> g_launches{0};
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

}  // namespace b200gs

using namespace b200gs;

extern "C" {

const char* b200gs_last_error(void) { return g_error; }
int b200gs_version(void) { return 237; }
int64_t b200gs_launch_count(void) { return (int64_t)g_launches.load(std::memory_order_relaxed); }

int b200gs_ipc_alloc(size_t bytes, void** dev_ptr, unsigned char* handle64) {
    B200GS_CHECK_ARG(dev_ptr != nullptr && handle64 != nullptr && bytes > 0, "bad arguments");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle is 64 bytes");
    void* p = nullptr;
    B200GS_CUDA(cudaMalloc(&p, bytes));
    cudaIpcMemHandle_t h;
    cudaError_t e = cudaIpcGetMemHandle(&h, p);
    if (e != cudaSuccess) {
        cudaFree(p);
        set_error("b200gs_ipc_alloc: cudaIpcGetMemHandle failed: %s", cudaGetErrorString(e));
        return B200GS_ECUDA;
    }
    memcpy(handle64, &h, 64);
    *dev_ptr = p;
    return B200GS_OK;
}

int b200gs_ipc_open(const unsigned char* handle64, void** dev_ptr) {
    B200GS_CHECK_ARG(dev_ptr != nullptr && handle64 != nullptr, "bad arguments");
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, 64);
    B200GS_CUDA(cudaIpcOpenMemHandle(dev_ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return B200GS_OK;
}

int b200gs_ipc_close(void* dev_ptr) {
    if (dev_ptr) B200GS_CUDA(cudaIpcCloseMemHandle(dev_ptr));
    return B200GS_OK;
}

int b200gs_ipc_free(void* dev_ptr) {
    if (dev_ptr) B200GS_CUDA(cudaFree(dev_ptr));
    return B200GS_OK;
}

}  // extern "C"
