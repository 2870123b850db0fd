// subenv.cpp -- the device source of the per-env wrapper chains (gym_b200/csrc/subenv.cuh), compiled for the CPU.
//
// TEST INFRASTRUCTURE: runs subenv_step_env / subenv_reset_env -- the code subenv_step_kernel and subenv_reset_kernel
// run per thread -- for every env in a loop, so that tests/test_subenv_cpu.py can compare the chain with the numpy
// restatement (oracle/subenv_chain.py) without a GPU.  What it does not run is nvcc's code generation; the GPU suite
// (tests/test_gpu_subenv.py) covers that.
#include "cuda_shim.h"

#include "../../gym_b200/csrc/subenv.cuh"

static bgym::SubenvArgs args(const int32_t *op, int32_t raw_reward_type, int32_t int_reward_on_fall, const double *p0,
                             const double *p1, int num_stages,
                             int D, int64_t n, double *obs_stats, double *rew_stats, float *ep_return,
                             int32_t *ep_length) {
    bgym::SubenvArgs a{};
    a.num_stages = num_stages;
    for (int s = 0; s < num_stages; s++) {
        a.op[s] = op[s];
        a.p0[s] = p0[s];
        a.p1[s] = p1[s];
    }
    a.raw_reward_type = raw_reward_type;
    a.int_reward_on_fall = int_reward_on_fall;
    a.D = D;
    a.n = n;
    a.obs_stats = obs_stats;
    a.rew_stats = rew_stats;
    a.ep_return = ep_return;
    a.ep_length = ep_length;
    return a;
}

extern "C" {

void hs_subenv_step(const int32_t *op, int32_t raw_reward_type, int32_t int_reward_on_fall, const double *p0,
                    const double *p1, int num_stages, int D,
                    int64_t n, double *obs_stats, double *rew_stats, float *ep_return, int32_t *ep_length, float *obs,
                    double *reward, const uint8_t *term, const uint8_t *trunc, float *fin, double *fin64, float *ep_r,
                    int32_t *ep_l) {
    const bgym::SubenvArgs a = args(op, raw_reward_type, int_reward_on_fall, p0, p1, num_stages, D, n, obs_stats,
                                    rew_stats, ep_return, ep_length);
    for (int64_t i = 0; i < n; i++) bgym::subenv_step_env(a, i, obs, reward, term, trunc, fin, fin, fin64, ep_r, ep_l);
}

void hs_subenv_reset(const int32_t *op, int32_t raw_reward_type, int32_t int_reward_on_fall, const double *p0,
                     const double *p1, int num_stages, int D,
                     int64_t n, double *obs_stats, double *rew_stats, float *ep_return, int32_t *ep_length, float *obs) {
    const bgym::SubenvArgs a = args(op, raw_reward_type, int_reward_on_fall, p0, p1, num_stages, D, n, obs_stats,
                                    rew_stats, ep_return, ep_length);
    for (int64_t i = 0; i < n; i++) bgym::subenv_reset_env(a, i, obs);
}

void hs_clip(const float *x, float *out, int64_t total, float lo, float hi) {
    for (int64_t e = 0; e < total; e++) out[e] = bgym::np_clipf(x[e], lo, hi);
}

}  // extern "C"
