// Shared helpers for the sm_90a kernels of libcubemap_b200.so.
#pragma once
#include <cuda_runtime.h>
#include <algorithm>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <vector>
#include "../../include/cubemap_b200.h"

namespace cslam {

void set_error(const char* fmt, ...);   // thread-local message behind cslam_last_error()

#define CSLAM_CUDA(expr)                                                                        \
    do {                                                                                        \
        cudaError_t _e = (expr);                                                                \
        if (_e != cudaSuccess) {                                                                \
            cslam::set_error("%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
            return CSLAM_E_CUDA;                                                                \
        }                                                                                       \
    } while (0)

static inline int round_up(int v, int m) { return (v + m - 1) / m * m; }
static inline int cdiv(int a, int b) { return (a + b - 1) / b; }
static inline int pow2_at_least(int n) { int p = 1; while (p < n) p <<= 1; return p; }   // sizes of the block-wide bitonic sorts

// Device buffer of `count` elements (at least one) owned by a handle: it goes onto `owned`, which the handle's destroy frees. zero: cleared once.
template <class T>
static int dev_alloc(std::vector<void*>& owned, T** p, size_t count, bool zero) {
    void* q = nullptr;
    const size_t bytes = std::max<size_t>(count, 1) * sizeof(T);
    CSLAM_CUDA(cudaMalloc(&q, bytes));
    owned.push_back(q);
    if (zero) CSLAM_CUDA(cudaMemset(q, 0, bytes));
    *p = (T*)q;
    return 0;
}
// Page-locked host buffer of `count` elements (at least one) owned by a handle: it goes onto `pinned`, which the handle's destroy frees.
template <class T>
static int pinned_alloc(std::vector<void*>& pinned, T** p, size_t count) {
    void* q = nullptr;
    CSLAM_CUDA(cudaMallocHost(&q, std::max<size_t>(count, 1) * sizeof(T)));
    pinned.push_back(q);
    *p = (T*)q;
    return 0;
}

// Device memory of a handle's single calls (staged inputs, outputs, scratch), carved from chunks the handle keeps across calls: cudaMalloc /
// cudaFree per call would cost more than many of the calls themselves. Pieces are 256-byte aligned and go to the first chunk with room; a new
// chunk is max(request, minimum) bytes, so a call sequence of fixed shape lands on the same pieces every time and stops allocating after its
// first call. Rules:
// - Only public entry points call reset(), and only on entry, before anything is taken. All of a handle's work is ordered by its one
//   stream, so a piece is reused only by work enqueued after the work that last used it.
// - A function that another entry point calls never resets: a host form that called a resetting _dev form would give its staged inputs
//   away to the _dev form's scratch.
// - Work on arena memory runs on the handle's stream, or on streams forked from it (the front end's lanes) if they are joined back into
//   it and the entry point synchronises the handle's stream before it returns. Every fill or copy into arena memory is cudaMemsetAsync /
//   cudaMemcpyAsync on one of those streams: a legacy-stream cudaMemset / cudaMemcpy does not order against a non-blocking stream.
// - Chunks are freed only by the destructor: cudaFree synchronises the device, and a _dev call may still be in flight.
class DevArena {
  public:
    DevArena() = default;
    DevArena(const DevArena&) = delete;
    DevArena& operator=(const DevArena&) = delete;
    ~DevArena() { for (auto& c : chunks) cudaFree(c.p); }
    void reset() { for (auto& c : chunks) c.used = 0; }
    // `count` elements (at least one); zero: cleared on the stream
    template <class T>
    int take(T** p, size_t count, bool zero = false) {
        const size_t bytes = (std::max<size_t>(count, 1) * sizeof(T) + 255) & ~(size_t)255;
        char* q = nullptr;
        for (auto& c : chunks) if (c.size - c.used >= bytes) { q = c.p + c.used; c.used += bytes; break; }
        if (!q) {
            Chunk c; c.size = std::max(bytes, minBytes); c.used = bytes;
            CSLAM_CUDA(cudaMalloc((void**)&c.p, c.size));
            chunks.push_back(c); q = c.p;
        }
        if (zero) CSLAM_CUDA(cudaMemsetAsync(q, 0, bytes, stream));
        *p = (T*)q;
        return 0;
    }
    // take + one host-to-device copy of `count` elements
    template <class T>
    int upload(const T** p, const T* host, size_t count) {
        T* q = nullptr;
        const int rc = take(&q, count);
        if (rc) return rc;
        if (count) CSLAM_CUDA(cudaMemcpyAsync(q, host, count * sizeof(T), cudaMemcpyHostToDevice, stream));
        *p = q;
        return 0;
    }

  private:
    friend struct Handle;   // Handle::open gives the arena its stream and minimum chunk
    struct Chunk { char* p; size_t size, used; };
    std::vector<Chunk> chunks;
    cudaStream_t stream = nullptr;
    size_t minBytes = 0;
};

// What every handle of the C ABI owns, with one definition of its lifecycle (capi_common.cu). The handle structs derive from it.
// - open(): check the device, create the handle's non-blocking stream (all of its work is ordered by it), give the arena that stream and
//   its minimum chunk, and, for handles whose kernels report overflow, allocate the zeroed device error flag and its pinned host copy.
// - sync(): wait for the stream; a set error flag is cleared and reported once, with the handle's message, as the code the kernel wrote.
//   Every synchronous host entry point ends with it.
// - destroy_handle(): the one way a handle ends, also on the failure paths of its create.
struct Handle {
    int device = 0;
    cudaStream_t stream = nullptr;
    DevArena arena;                 // staging of the host entry points
    std::vector<void*> owned;       // dev_alloc
    std::vector<void*> pinned;      // pinned_alloc
    int64_t launches = 0;
    int* errFlag = nullptr;         // device; CSLAM_E_* of the first overflow since the last sync(); nullptr: the handle has none
    int* errHost = nullptr;         // pinned copy of *errFlag

    Handle() = default;
    Handle(const Handle&) = delete;
    Handle& operator=(const Handle&) = delete;
    ~Handle();   // frees owned, pinned, the arena's chunks and the stream: only through destroy_handle, which has waited for the stream
    int open(int device, size_t arenaMinChunk, bool wantErrFlag);
    int sync(const char* overflowMessage = nullptr);
};

// Waits for the handle's stream, then deletes it. The wait cannot live in ~Handle: a derived handle's members are destroyed before the
// base destructor runs, and a derived destructor may free what the stream's work still uses.
template <class H>
static void destroy_handle(H* h) {
    if (!h) return;
    if (h->stream) {   // nothing is allocated before open() has created the stream
        cudaSetDevice(h->device);
        cudaStreamSynchronize(h->stream);
    }
    delete h;
}

// Optional per-kernel timing of a handle (cslam_*_set_timing / cslam_*_get_timing): record() puts an event on the stream before each
// launch, and collect() adds the time from every event to the next one to the kind of the earlier event. A handle records END after its
// last launch; the interval that starts there (up to the next call's first launch) belongs to no kernel and is not counted.
struct KernelTimer {
    static const int END = -1, MAX_KINDS = 16;
    KernelTimer() = default;
    KernelTimer(const KernelTimer&) = delete;
    KernelTimer& operator=(const KernelTimer&) = delete;
    ~KernelTimer() { for (cudaEvent_t e : ev) cudaEventDestroy(e); }
    bool on() const { return enabled; }
    // the first enable creates `capacity` events on the current device (records beyond them are dropped); every call clears the totals
    int enable(bool en, int capacity) {
        if (en && ev.empty()) {
            ev.resize(capacity); evKind.resize(capacity);
            for (auto& e : ev) CSLAM_CUDA(cudaEventCreate(&e));
        }
        enabled = en; used = 0;
        for (int i = 0; i < MAX_KINDS; i++) { ms[i] = 0; count[i] = 0; }
        return CSLAM_OK;
    }
    void record(cudaStream_t st, int kind) {
        if (!enabled || used >= (int)ev.size()) return;
        cudaEventRecord(ev[used], st);
        evKind[used++] = kind;
    }
    void collect() {   // after the stream has been synchronised
        for (int i = 0; i + 1 < used; i++) {
            float t = 0;
            if (evKind[i] != END && cudaEventElapsedTime(&t, ev[i], ev[i + 1]) == cudaSuccess) { ms[evKind[i]] += t; count[evKind[i]]++; }
        }
        used = 0;
    }
    int get(int kind, int nkinds, const char* const* names, const char** name, double* msOut, int64_t* countOut) const {
        if (kind < 0 || kind >= nkinds) return CSLAM_E_BADARG;
        *name = names[kind]; *msOut = ms[kind]; *countOut = count[kind];
        return CSLAM_OK;
    }

  private:
    bool enabled = false;
    std::vector<cudaEvent_t> ev; std::vector<int> evKind; int used = 0;
    double ms[MAX_KINDS] = {0}; int64_t count[MAX_KINDS] = {0};
};

// ---------------------------------------------------------------------------------------------------------
// Device math with pinned rounding. The CPU path these must match bit-for-bit is specified without FMA
// contraction (oracle/cvprim.h); nvcc contracts a*b+c by default, so every fp32 step is spelled out.

// cv::fastAtan2 (scalar path), degrees.
__device__ __forceinline__ float fast_atan2_deg(float y, float x) {
    const float s = (float)(180.0 / 3.14159265358979323846);
    const float p1 = 0.9997878412794807f * s, p3 = -0.3258083974640975f * s;
    const float p5 = 0.1555786518463281f * s, p7 = -0.04432655554792128f * s;
    const float eps = 2.220446049250313e-16f;   // (float)DBL_EPSILON
    float ax = fabsf(x), ay = fabsf(y), a, c, c2;
    if (ax >= ay) {
        c = __fdiv_rn(ay, __fadd_rn(ax, eps));
        c2 = __fmul_rn(c, c);
        a = __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c);
    } else {
        c = __fdiv_rn(ax, __fadd_rn(ay, eps));
        c2 = __fmul_rn(c, c);
        a = __fsub_rn(90.f, __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c));
    }
    if (x < 0) a = __fsub_rn(180.f, a);
    if (y < 0) a = __fsub_rn(360.f, a);
    return a;
}

// det_sincos (DESIGN.md): fp64 Cody-Waite reduction by pi/2 + fdlibm kernel polynomials, only IEEE mul/fma,
// rounded once to fp32. fp64 mul/fma are bit-identical on host and device, so this equals the CPU definition.
__device__ __forceinline__ void det_sincosf(float xf, float* s_out, float* c_out) {
    const double x = (double)xf;
    const double kd = rint(__dmul_rn(x, 0.63661977236758134308));
    const int k = (int)kd;
    double r = __fma_rn(-kd, 1.57079632679489655800e+00, x);
    r = __fma_rn(-kd, 6.12323399573676603587e-17, r);
    const double r2 = __dmul_rn(r, r);
    double ps = 1.58969099521155010221e-10;
    ps = __fma_rn(ps, r2, -2.50507602534068634195e-08);
    ps = __fma_rn(ps, r2, 2.75573137070700676789e-06);
    ps = __fma_rn(ps, r2, -1.98412698298579493134e-04);
    ps = __fma_rn(ps, r2, 8.33333333332248946124e-03);
    ps = __fma_rn(ps, r2, -1.66666666666666324348e-01);
    const double sn = __fma_rn(__dmul_rn(r, r2), ps, r);
    double pc = -1.13596475577881948265e-11;
    pc = __fma_rn(pc, r2, 2.08757232129817482790e-09);
    pc = __fma_rn(pc, r2, -2.75573143513906633035e-07);
    pc = __fma_rn(pc, r2, 2.48015872894767294178e-05);
    pc = __fma_rn(pc, r2, -1.38888888888741095749e-03);
    pc = __fma_rn(pc, r2, 4.16666666666666019037e-02);
    const double cs = __fma_rn(__dmul_rn(r2, r2), pc, __fma_rn(-0.5, r2, 1.0));
    double sv, cv;
    switch (k & 3) {
        case 0: sv = sn; cv = cs; break;
        case 1: sv = cs; cv = -sn; break;
        case 2: sv = -sn; cv = -cs; break;
        default: sv = -cs; cv = sn; break;
    }
    *s_out = (float)sv;
    *c_out = (float)cv;
}

__device__ __forceinline__ int reflect101(int p, int n) {
    if (p < 0) p = -p;
    if (p >= n) p = 2 * (n - 1) - p;
    return p;
}

}  // namespace cslam
