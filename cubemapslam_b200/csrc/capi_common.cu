// Error reporting and library-wide entry points of libcubemap_b200.so.
#include "common.cuh"

namespace cslam {
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
int check_device(int device) {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) { set_error("no CUDA device (this library has no CPU fallback)"); return CSLAM_E_NODEVICE; }
    if (device < 0 || device >= ndev) { set_error("device %d out of range (%d devices)", device, ndev); return CSLAM_E_BADARG; }
    CSLAM_CUDA(cudaSetDevice(device));
    return CSLAM_OK;
}
}  // namespace cslam

extern "C" const char* cslam_last_error(void) { return cslam::g_err; }
extern "C" int cslam_version(void) { return 100; }
extern "C" int cslam_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
    return n;
}
