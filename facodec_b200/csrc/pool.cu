// Slot <-> lane moves of the stream pools (fac_codes_pool_*, fac_vc_pool_*, fac_dec_pool_*): each lane of a batch reads or
// writes its own session's buffer through a pointer table passed as a kernel parameter, so a step needs no host-to-device
// copy.  Each lane moves its own word count (a decode pool's lanes end at their own last frame).  The same kernel, wider,
// moves exported and imported session state between slots and state payloads.
#include "common.cuh"
#include "kernels.h"

namespace fac {

template <int N>
__global__ void lane_copy_kernel(const __grid_constant__ LaneCopyParamsN<N> p) {
    const int b = blockIdx.y;
    if (b >= p.n) return;
    const uint32_t* src = p.src[b];
    uint32_t* dst = p.dst[b];
    const long long words = p.words[b];
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < words; i += (long long)gridDim.x * blockDim.x)
        dst[i] = src[i];
}

template <int N>
cudaError_t lane_copy_launch(const LaneCopyParamsN<N>& p, cudaStream_t st) {
    if (p.n <= 0) return cudaSuccess;
    if (p.n > N) return cudaErrorInvalidValue;
    long long most = 0;
    for (int b = 0; b < p.n; ++b) most = p.words[b] > most ? p.words[b] : most;
    if (most <= 0) return cudaSuccess;
    long long blocks = (most + 255) / 256;
    if (blocks > 64) blocks = 64;
    lane_copy_kernel<N><<<dim3((unsigned)blocks, p.n), 256, 0, st>>>(p);
    return cudaGetLastError();
}

cudaError_t launch_lane_copy(const LaneCopyParamsN<kLaneMax>& p, cudaStream_t st) { return lane_copy_launch(p, st); }
cudaError_t launch_lane_copy(const LaneCopyParamsN<kMoveLanes>& p, cudaStream_t st) { return lane_copy_launch(p, st); }

}  // namespace fac
