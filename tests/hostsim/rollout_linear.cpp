// rollout_linear.cpp -- the per-env driver of rollout_linear_kernel, compiled for the CPU.
//
// TEST INFRASTRUCTURE (never shipped, never imported by gym_b200/): includes gym_b200/csrc/per_env.cuh through
// tests/hostsim/cuda_shim.h (by way of rollout.cpp, whose batch layout and reset / step entry points it shares) and runs
// rollout_linear_env for every env, and Env<KIND>::observe of every env's state.  tests/test_rollout_linear_cpu.py
// compares one linear-policy rollout with a numpy restatement of the policy and T kernel-A steps of the same batch.
// The argument set-up copies b200gym_rollout_linear.
#include "rollout.cpp"

extern "C" {

// one b200gym_rollout_linear launch of T steps; returns NULL: per-step outputs, else the summary (actions ... final_obs
// unused) -> 0 (-1: bad kind)
int64_t hs_rol_rollout(const Batch *B, const float *weight, const float *bias, int per_env, int32_t T,
                       void *actions_out, float *obs, double *reward, uint8_t *term, uint8_t *trunc, float *final_obs,
                       double *returns, int32_t *lengths, uint8_t *ended, float *last_obs) {
    unsigned long long invalid = 0, seen = 0;
    const bool summary = returns != nullptr;
    const StepArgs a = summary ? args_of(*B, &invalid, &seen, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr)
                               : args_of(*B, &invalid, &seen, actions_out, obs, reward, term, trunc, final_obs);
    return dispatch(B->kind, B->kind == B200GYM_CARTPOLE || B->kind == B200GYM_MOUNTAINCAR || B->kind == B200GYM_ACROBOT
                                 ? B200GYM_ACT_I64 : B200GYM_ACT_F32,
                    [&](auto k, auto *) -> int64_t {
                        constexpr int KIND = decltype(k)::value;
                        const int64_t K = linear_logit_count<KIND>(), D = bgym::Env<KIND>::D;
                        const LinearPolicyArgs p{weight, bias, per_env ? K * D : 0, per_env ? K : 0, returns, lengths,
                                                 ended};
                        for (int64_t i = 0; i < a.n; i++) {
                            if (summary) rollout_linear_env<KIND, true>(a, i, T, last_obs, p);
                            else rollout_linear_env<KIND, false>(a, i, T, last_obs, p);
                        }
                        return invalid ? -2 : 0;
                    });
}

// Env<KIND>::observe of every env's state into obs [n][obs_dim] -> 0 (-1: bad kind)
int64_t hs_rol_observe(const Batch *B, float *obs) {
    return dispatch(B->kind, B->kind == B200GYM_CARTPOLE || B->kind == B200GYM_MOUNTAINCAR || B->kind == B200GYM_ACROBOT
                                 ? B200GYM_ACT_I64 : B200GYM_ACT_F32,
                    [&](auto k, auto *) -> int64_t {
                        using E = bgym::Env<decltype(k)::value>;
                        for (int64_t i = 0; i < B->n; i++) {
                            double s[E::S];
                            float o[E::D];
                            for (int j = 0; j < E::S; j++) s[j] = B->state[j * B->n + i];
                            E::observe(s, o);
                            for (int j = 0; j < E::D; j++) obs[i * E::D + j] = o[j];
                        }
                        return 0;
                    });
}

}  // extern "C"
