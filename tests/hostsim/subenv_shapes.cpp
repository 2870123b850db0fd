// subenv_shapes.cpp -- the reshaping wrapper chains and action stages of gym_b200/csrc/subenv.cuh, compiled for the CPU.
//
// TEST INFRASTRUCTURE: runs what subenv_step_kernel, subenv_reset_kernel and subenv_action_kernel run per thread --
// subenv_step_env_io / subenv_reset_env_io / subenv_action, with the widths and dtypes resolved by subenv_resolve as
// b200gym_subenv_set resolves them -- for every env in a loop, so that tests/test_subenv_shapes_cpu.py can compare them
// with the numpy restatement (oracle/subenv_shapes.py) without a GPU.
#include "cuda_shim.h"

#include "../../gym_b200/csrc/subenv.cuh"

struct HsState {
    double *obs_stats, *rew_stats;
    float *ep_return;
    int32_t *ep_length;
    void *history;
    int32_t *head;
    int64_t *t;
};

static bgym::SubenvArgs args(const int32_t *op, const double *p0, const double *p1, int num_stages,
                             int32_t raw_reward_type, int32_t int_reward_on_fall, int D, int64_t n, const HsState *st) {
    bgym::SubenvArgs a{};
    a.num_stages = num_stages;
    bool time_aware = false;
    for (int s = 0; s < num_stages; s++) {
        a.op[s] = op[s];
        a.p0[s] = p0[s];
        a.p1[s] = p1[s];
        time_aware |= op[s] == bgym::kSubTimeAware;
    }
    a.raw_reward_type = raw_reward_type;
    a.int_reward_on_fall = int_reward_on_fall;
    a.D = D;
    a.n = n;
    a.obs_stats = st->obs_stats;
    a.rew_stats = st->rew_stats;
    a.ep_return = st->ep_return;
    a.ep_length = st->ep_length;
    a.history = st->history;
    a.head = st->head;
    a.tstep = time_aware ? st->t : nullptr;
    bgym::subenv_resolve(a);
    return a;
}

extern "C" {

int hs_shape_width(const int32_t *op, const double *p0, int num_stages, int D, int32_t *out_f64) {
    bgym::SubenvArgs a{};
    a.num_stages = num_stages;
    for (int s = 0; s < num_stages; s++) {
        a.op[s] = op[s];
        a.p0[s] = p0[s];
    }
    a.D = D;
    bgym::subenv_resolve(a);
    *out_f64 = a.out_f64;
    return a.W;
}

void hs_shape_step(const int32_t *op, const double *p0, const double *p1, int num_stages, int32_t raw_reward_type,
                   int32_t int_reward_on_fall, int D, int64_t n, const HsState *st, const float *obs_in,
                   float *obs_out, double *reward, const uint8_t *term, const uint8_t *trunc, const float *fin_in,
                   float *fin_out, double *fin64, float *ep_r, int32_t *ep_l) {
    const bgym::SubenvArgs a = args(op, p0, p1, num_stages, raw_reward_type, int_reward_on_fall, D, n, st);
    for (int64_t i = 0; i < n; i++)
        bgym::subenv_step_env_io(a, i, obs_in, obs_out, reward, term, trunc, fin_in, fin_out, fin64, ep_r, ep_l);
}

void hs_shape_reset(const int32_t *op, const double *p0, const double *p1, int num_stages, int32_t raw_reward_type,
                    int32_t int_reward_on_fall, int D, int64_t n, const HsState *st, const float *obs_in,
                    float *obs_out) {
    const bgym::SubenvArgs a = args(op, p0, p1, num_stages, raw_reward_type, int_reward_on_fall, D, n, st);
    for (int64_t i = 0; i < n; i++) bgym::subenv_reset_env_io(a, i, obs_in, obs_out);
}

// b: num, op[2], lo[2][4], hi[2][4], amin[2][4], amax[2][4] as SubenvActions lays them out
void hs_actions(const bgym::SubenvActions *b, const float *in, float *out, int64_t total, int A) {
    for (int64_t e = 0; e < total; e++) out[e] = bgym::subenv_action(*b, (int)(e % A), in[e]);
}

}  // extern "C"
