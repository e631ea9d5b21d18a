// Shared host/device pieces of the optimizer translation units (ba.cu: LocalBundleAdjustment, pose_opt.cu: PoseOptimization).
#pragma once
#include <algorithm>
#include <vector>
#include "area_table.cuh"
#include "ba_math.cuh"
#include "common.cuh"

typedef void* nccl_comm_t;

struct cslam_optimizer : cslam::Handle {
    nccl_comm_t comm = nullptr; int rank = 0, nranks = 1;
    double* h_scal = nullptr;   // pinned, 16 doubles
    // host scratch of cslam_local_ba, kept across calls (fresh multi-megabyte vectors cost page faults on every call)
    struct HostScratch { std::vector<int> lmStart, perm, eMP, eKF, fill, peStart, peList, kfOfQ; std::vector<double> X; } hs;
    cslam::KernelTimer timer;   // optional per-kernel timing (cslam_optimizer_set_timing); LM trials then run eagerly instead of as a graph
    // one-shot NVLink all-reduce of the reduced camera system (multi-GPU LocalBA): peer views of every rank's exchange buffer
    struct Peer { void* base = nullptr; bool mine = false; };
    std::vector<Peer> peers; size_t xchgBytes = 0; uint32_t epoch = 0, epoch2 = 0; bool oneShot = false;
    ~cslam_optimizer();   // ba.cu: the peers' exchange buffers and the NCCL communicator
};

namespace cslam {

#ifdef __CUDACC__
// fixed-shape (deterministic) block sum; result valid in thread 0. sh: >= 32 doubles
__device__ __forceinline__ double block_sum(double v, double* sh) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (lane == 0) sh[w] = v;
    __syncthreads();
    double r = 0;
    if (w == 0) {
        r = lane < (blockDim.x >> 5) ? sh[lane] : 0.0;
#pragma unroll
        for (int o = 16; o; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
    }
    __syncthreads();
    return r;
}
#endif

}  // namespace cslam
