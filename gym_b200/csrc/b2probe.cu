// b2probe.cu -- the device side of b200gym_selftest_box2d (b200gym.cu): the Box2D building blocks of b2lite.cuh on
// packed records (b2probe.cuh), one thread per record.
//
// A translation unit of its own: the probe calls the solver's non-inlined device functions (collide_edge_polygon,
// gjk_distance, time_of_impact, ...), and a new caller in b200gym.cu's module would let ptxas compile those functions,
// and so the step kernels that call them, differently.  Here they get their own copies, compiled from the same source
// with the same flags, and b200gym.cu's kernels stay as they are.  The module also has its own copy of the task
// constants (lunar::kC, walker::kC), loaded with the same host code as b200gym_create loads the engine's.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdint>
#include <cstring>
#include <type_traits>

// The headers define the solver's non-inlined functions and the constants at namespace scope, as b200gym.cu includes
// them too: inside an unnamed namespace this module's copies keep to this module
namespace {

#include "box2d_consts.h"
#include "b2probe.cuh"

constexpr int kProbeThreads = 128;

__global__ void __launch_bounds__(kProbeThreads) selftest_box2d_kernel(int op, const float *in, int64_t n, float *out) {
    const int64_t i = (int64_t)blockIdx.x * kProbeThreads + threadIdx.x;
    if (i >= n) return;
    b2probe::probe_case(op, in + i * b2probe::kProbeWords, out + i * b2probe::kProbeWords);
}

}  // namespace

// called by b200gym_selftest_box2d on the caller's device, after the arguments are checked
cudaError_t b2probe_launch(int op, const float *in_dev, int64_t n, float *out_dev, cudaStream_t stream) {
    lunar::Consts lc;
    walker::Consts wc;
    b2l_host::lunar_consts(lc);
    b2l_host::walker_consts(wc);
    cudaError_t e = cudaMemcpyToSymbol(lunar::kC, &lc, sizeof lc);
    if (e == cudaSuccess) e = cudaMemcpyToSymbol(walker::kC, &wc, sizeof wc);
    if (e != cudaSuccess) return e;
    selftest_box2d_kernel<<<(unsigned)((n + kProbeThreads - 1) / kProbeThreads), kProbeThreads, 0, stream>>>(op, in_dev, n,
                                                                                                           out_dev);
    return cudaGetLastError();
}

int b2probe_num_ops() { return b2probe::PROBE_NUM_OPS; }
