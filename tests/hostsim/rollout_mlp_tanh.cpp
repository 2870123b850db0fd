// rollout_mlp_tanh.cpp -- the tanh instantiations of the per-env drivers of rollout_mlp_kernel and
// rollout_mlp_noisy_kernel, compiled for the CPU.
//
// TEST INFRASTRUCTURE (never shipped, never imported by gym_b200/): rollout_mlp.cpp and rollout_mlp_noisy.cpp with
// ACT = B200GYM_MLP_TANH, so mlp_tanh is the host C library's tanhf.  tests/test_rollout_mlp_tanh_cpu.py compares them
// with the numpy restatements of test_rollout_mlp_cpu.py / test_rollout_mlp_noisy_cpu.py, their activation swapped
// for that same tanhf called through ctypes.
#include "rollout.cpp"

extern "C" {

// hs_mlp_rollout (rollout_mlp.cpp) with the tanh activation
int64_t hs_mlp_tanh_rollout(const Batch *B, const float *params, int per_env, int h1, int h2, int32_t T,
                            void *actions_out, float *obs, double *reward, uint8_t *term, uint8_t *trunc,
                            float *final_obs, double *returns, int32_t *lengths, uint8_t *ended, float *last_obs) {
    unsigned long long invalid = 0, seen = 0;
    const bool summary = returns != nullptr;
    const StepArgs a = summary ? args_of(*B, &invalid, &seen, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr)
                               : args_of(*B, &invalid, &seen, actions_out, obs, reward, term, trunc, final_obs);
    return dispatch(B->kind, B->kind == B200GYM_CARTPOLE || B->kind == B200GYM_MOUNTAINCAR || B->kind == B200GYM_ACROBOT
                                 ? B200GYM_ACT_I64 : B200GYM_ACT_F32,
                    [&](auto k, auto *) -> int64_t {
                        constexpr int KIND = decltype(k)::value, ACT = B200GYM_MLP_TANH;
                        constexpr int K = linear_logit_count<KIND>(), D = bgym::Env<KIND>::D;
                        const int64_t P = mlp_param_count<K, D>(h1, h2);
                        const bool vec = h1 % 4 == 0 && (!per_env || P % 4 == 0);
                        const MlpPolicyArgs p{params, per_env ? P : 0, h1, h2, vec ? 1 : 0, returns, lengths, ended};
                        for (int64_t i = 0; i < a.n; i++) {
                            const float *w = params + i * p.stride;
                            if (per_env) {
                                if (summary) rollout_mlp_env<KIND, true, true, ACT>(a, i, T, last_obs, w, p);
                                else rollout_mlp_env<KIND, false, true, ACT>(a, i, T, last_obs, w, p);
                            } else {
                                if (summary) rollout_mlp_env<KIND, true, false, ACT>(a, i, T, last_obs, w, p);
                                else rollout_mlp_env<KIND, false, false, ACT>(a, i, T, last_obs, w, p);
                            }
                        }
                        return invalid ? -2 : 0;
                    });
}

// hs_mlp_noisy_rollout (rollout_mlp_noisy.cpp) with the tanh activation
int64_t hs_mlp_noisy_tanh_rollout(const Batch *B, const float *params, int per_env, int h1, int h2, int32_t T,
                                  const float *noise, float *outputs, void *actions_out, float *obs, double *reward,
                                  uint8_t *term, uint8_t *trunc, float *final_obs, float *last_obs) {
    unsigned long long invalid = 0, seen = 0;
    const StepArgs a = args_of(*B, &invalid, &seen, actions_out, obs, reward, term, trunc, final_obs);
    return dispatch(B->kind, B->kind == B200GYM_CARTPOLE || B->kind == B200GYM_MOUNTAINCAR || B->kind == B200GYM_ACROBOT
                                 ? B200GYM_ACT_I64 : B200GYM_ACT_F32,
                    [&](auto k, auto *) -> int64_t {
                        constexpr int KIND = decltype(k)::value, ACT = B200GYM_MLP_TANH;
                        constexpr int K = linear_logit_count<KIND>(), D = bgym::Env<KIND>::D;
                        const int64_t P = mlp_param_count<K, D>(h1, h2);
                        const bool vec = h1 % 4 == 0 && (!per_env || P % 4 == 0);
                        const MlpNoisyArgs p{{params, per_env ? P : 0, h1, h2, vec ? 1 : 0, nullptr, nullptr, nullptr},
                                             noise, outputs};
                        for (int64_t i = 0; i < a.n; i++) {
                            const float *w = params + i * p.mlp.stride;
                            if (per_env) rollout_mlp_noisy_env<KIND, true, ACT>(a, i, T, last_obs, w, p);
                            else rollout_mlp_noisy_env<KIND, false, ACT>(a, i, T, last_obs, w, p);
                        }
                        return invalid ? -2 : 0;
                    });
}

}  // extern "C"
