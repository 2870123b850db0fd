// rollout_norm.cpp -- the per-env drivers of rollout_mlp_noisy_norm_kernel, rollout_actor_critic_norm_kernel and
// gae_scaled_kernel, compiled for the CPU.
//
// TEST INFRASTRUCTURE (never shipped, never imported by gym_b200/): includes gym_b200/csrc/per_env.cuh through
// tests/hostsim/cuda_shim.h (by way of rollout.cpp, whose batch layout and reset / step entry points it shares).  The
// statistics are staged as the kernels stage them, mean[D] and sd[D] = norm_sd(var[D], eps), once per call; the nets
// are read where the kernels read their shared-memory copies.  tests/test_rollout_norm_cpu.py compares the drivers with
// a numpy restatement (float64 normalisation, float32 MLP), and with the drivers without normalisation.
#include "rollout.cpp"

extern "C" {

// one b200gym_rollout_mlp_noisy_norm launch of T steps with one shared policy (h2 = 0: one hidden layer; act: a
// b200gym_mlp_activation), noise and outputs [T][n][K]; clip +inf: none -> 0 (-1: bad kind)
int64_t hs_mlp_noisy_norm_rollout(const Batch *B, const float *params, int h1, int h2, int act, int32_t T,
                                  const float *noise, float *outputs, void *actions_out, float *obs, double *reward,
                                  uint8_t *term, uint8_t *trunc, float *final_obs, float *last_obs, const double *mean,
                                  const double *var, double eps, float clip) {
    unsigned long long invalid = 0, seen = 0;
    const StepArgs a = args_of(*B, &invalid, &seen, actions_out, obs, reward, term, trunc, final_obs);
    const bool vec = h1 % 4 == 0;
    const MlpNoisyArgs p{{params, 0, h1, h2, vec ? 1 : 0, nullptr, nullptr, nullptr}, noise, outputs};
    double sd[24];
    return dispatch(B->kind, B->kind == B200GYM_CARTPOLE || B->kind == B200GYM_MOUNTAINCAR || B->kind == B200GYM_ACROBOT
                                 ? B200GYM_ACT_I64 : B200GYM_ACT_F32,
                    [&](auto k, auto *) -> int64_t {
                        constexpr int KIND = decltype(k)::value;
                        for (int c = 0; c < bgym::Env<KIND>::D; c++) sd[c] = norm_sd(var[c], eps);
                        for (int64_t i = 0; i < a.n; i++) {
                            if (act == B200GYM_MLP_TANH)
                                rollout_mlp_noisy_norm_env<KIND, B200GYM_MLP_TANH>(a, i, T, last_obs, params, p, mean,
                                                                                   sd, clip);
                            else rollout_mlp_noisy_norm_env<KIND, B200GYM_MLP_RELU>(a, i, T, last_obs, params, p, mean,
                                                                                    sd, clip);
                        }
                        return invalid ? -2 : 0;
                    });
}

// one b200gym_rollout_actor_critic_norm call with normalised observations: the rollout launch, then the GAE launch,
// gae_scaled_env when ret_var is not null (clip_r +inf: none), gae_env otherwise
int64_t hs_actor_critic_norm_rollout(const Batch *B, const float *actor, const float *critic, int h1, int h2, int act,
                                     int32_t T, const float *noise, float *outputs, void *actions_out, float *obs,
                                     double *reward, uint8_t *term, uint8_t *trunc, float *final_obs, float *values,
                                     float *advantages, float g, float gl, float *last_obs, const double *mean,
                                     const double *var, double eps, float clip, const double *ret_var, float clip_r) {
    unsigned long long invalid = 0, seen = 0;
    const StepArgs a = args_of(*B, &invalid, &seen, actions_out, obs, reward, term, trunc, final_obs);
    const bool vec = h1 % 4 == 0;
    const ActorCriticArgs p{{{actor, 0, h1, h2, vec ? 1 : 0, nullptr, nullptr, nullptr}, noise, outputs}, critic, values,
                            advantages};
    double sd[24];
    const int64_t rc = dispatch(
        B->kind, B->kind == B200GYM_CARTPOLE || B->kind == B200GYM_MOUNTAINCAR || B->kind == B200GYM_ACROBOT
                     ? B200GYM_ACT_I64 : B200GYM_ACT_F32,
        [&](auto k, auto *) -> int64_t {
            constexpr int KIND = decltype(k)::value;
            for (int c = 0; c < bgym::Env<KIND>::D; c++) sd[c] = norm_sd(var[c], eps);
            for (int64_t i = 0; i < a.n; i++) {
                if (act == B200GYM_MLP_TANH)
                    rollout_actor_critic_norm_env<KIND, B200GYM_MLP_TANH>(a, i, T, last_obs, actor, critic, p, mean, sd,
                                                                          clip);
                else rollout_actor_critic_norm_env<KIND, B200GYM_MLP_RELU>(a, i, T, last_obs, actor, critic, p, mean,
                                                                           sd, clip);
            }
            return invalid ? -2 : 0;
        });
    if (rc) return rc;
    for (int64_t i = 0; i < a.n; i++) {
        if (ret_var) gae_scaled_env(i, a.n, T, g, gl, norm_sd(ret_var[0], eps), clip_r, reward, term, trunc, values,
                                    advantages);
        else gae_env(i, a.n, T, g, gl, reward, term, trunc, values, advantages);
    }
    return 0;
}

// gae_scaled_kernel's per-env work for every env of [T][n] rows, with sd = norm_sd(ret_var, eps)
void hs_gae_scaled(int64_t n, int32_t T, float g, float gl, double ret_var, double eps, float clip_r,
                   const double *reward, const uint8_t *term, const uint8_t *trunc, const float *values, float *adv) {
    const double sd = norm_sd(ret_var, eps);
    for (int64_t i = 0; i < n; i++) gae_scaled_env(i, n, T, g, gl, sd, clip_r, reward, term, trunc, values, adv);
}

// norm_obs_elem over m elements of one column's statistics
void hs_norm_elems(int64_t m, const float *o, double mean, double var, double eps, float clip, float *x) {
    const double sd = norm_sd(var, eps);
    for (int64_t k = 0; k < m; k++) x[k] = norm_obs_elem(o[k], mean, sd, clip);
}

}  // extern "C"
