// Error reporting, the handle lifecycle and library-wide entry points of libcubemap_b200.so.
#include "common.cuh"

namespace cslam {
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
// CSLAM_E_NODEVICE without a CUDA device (no CPU fallback), CSLAM_E_BADARG for a device out of range, else cudaSetDevice
static int check_device(int device) {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) { set_error("no CUDA device (this library has no CPU fallback)"); return CSLAM_E_NODEVICE; }
    if (device < 0 || device >= ndev) { set_error("device %d out of range (%d devices)", device, ndev); return CSLAM_E_BADARG; }
    CSLAM_CUDA(cudaSetDevice(device));
    return CSLAM_OK;
}

int Handle::open(int dev, size_t arenaMinChunk, bool wantErrFlag) {
    int rc = check_device(dev);
    if (rc) return rc;
    device = dev;
    CSLAM_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    arena.stream = stream; arena.minBytes = arenaMinChunk;
    if (wantErrFlag && ((rc = dev_alloc(owned, &errFlag, 1, true)) || (rc = pinned_alloc(pinned, &errHost, 1)))) return rc;
    return CSLAM_OK;
}

int Handle::sync(const char* overflowMessage) {
    CSLAM_CUDA(cudaSetDevice(device));
    if (errFlag) CSLAM_CUDA(cudaMemcpyAsync(errHost, errFlag, sizeof(int), cudaMemcpyDeviceToHost, stream));
    CSLAM_CUDA(cudaStreamSynchronize(stream));
    if (errFlag && *errHost) {
        const int code = *errHost;
        cudaMemsetAsync(errFlag, 0, sizeof(int), stream);
        set_error("%s", overflowMessage);
        return code;
    }
    return CSLAM_OK;
}

Handle::~Handle() {
    for (void* p : owned) cudaFree(p);
    for (void* p : pinned) cudaFreeHost(p);
    if (stream) cudaStreamDestroy(stream);
}
}  // namespace cslam

extern "C" const char* cslam_last_error(void) { return cslam::g_err; }
extern "C" int cslam_version(void) { return 101; }
extern "C" int cslam_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
    return n;
}
