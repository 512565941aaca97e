// api.cu -- version / error plumbing of the C-ABI (include/morl_b200.h).
#include <stdarg.h>
#include <string.h>

#include "common.cuh"

namespace morl {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int check_launch(const char* what) {
    cudaError_t e = cudaPeekAtLastError();
    if (e != cudaSuccess) {
        (void)cudaGetLastError();  // clear the sticky launch error so the next call starts clean
        set_error("%s: %s", what, cudaGetErrorString(e));
        return static_cast<int>(e);
    }
    return MORL_OK;
}

}  // namespace morl

extern "C" {

int morl_version(void) { return MORL_B200_VERSION; }

const char* morl_last_error(void) { return morl::g_err; }

int morl_device_sm_count(void) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) {
        (void)cudaGetLastError();
        morl::set_error("morl_device_sm_count: no CUDA device (%s)", cudaGetErrorString(e));
        return MORL_ERR_NO_DEVICE;
    }
    int n = 0;
    e = cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (e != cudaSuccess) {
        (void)cudaGetLastError();
        morl::set_error("morl_device_sm_count: %s", cudaGetErrorString(e));
        return MORL_ERR_NO_DEVICE;
    }
    return n;
}

}  // extern "C"
