// rollout_mlp_noisy.cpp -- the per-env driver of rollout_mlp_noisy_kernel, compiled for the CPU.
//
// TEST INFRASTRUCTURE (never shipped, never imported by gym_b200/): includes gym_b200/csrc/per_env.cuh through
// tests/hostsim/cuda_shim.h (by way of rollout.cpp, whose batch layout and reset / step entry points it shares) and runs
// rollout_mlp_noisy_env for every env.  A shared policy is read where the kernel reads its shared-memory copy, a per-env
// one row by row as the kernel reads device memory.  tests/test_rollout_mlp_noisy_cpu.py compares one noisy MLP-policy
// rollout with a numpy restatement of the policy plus the noise and T kernel-A steps of the same batch.  The argument
// set-up copies b200gym_rollout_mlp_noisy, the 16-byte rows (vec) included.
#include "rollout.cpp"

extern "C" {

// one b200gym_rollout_mlp_noisy launch of T steps (h2 = 0: one hidden layer), noise and outputs [T][n][K] -> 0 (-1:
// bad kind)
int64_t hs_mlp_noisy_rollout(const Batch *B, const float *params, int per_env, int h1, int h2, int32_t T,
                             const float *noise, float *outputs, void *actions_out, float *obs, double *reward,
                             uint8_t *term, uint8_t *trunc, float *final_obs, float *last_obs) {
    unsigned long long invalid = 0, seen = 0;
    const StepArgs a = args_of(*B, &invalid, &seen, actions_out, obs, reward, term, trunc, final_obs);
    return dispatch(B->kind, B->kind == B200GYM_CARTPOLE || B->kind == B200GYM_MOUNTAINCAR || B->kind == B200GYM_ACROBOT
                                 ? B200GYM_ACT_I64 : B200GYM_ACT_F32,
                    [&](auto k, auto *) -> int64_t {
                        constexpr int KIND = decltype(k)::value;
                        constexpr int K = linear_logit_count<KIND>(), D = bgym::Env<KIND>::D;
                        const int64_t P = mlp_param_count<K, D>(h1, h2);
                        const bool vec = h1 % 4 == 0 && (!per_env || P % 4 == 0);
                        const MlpNoisyArgs p{{params, per_env ? P : 0, h1, h2, vec ? 1 : 0, nullptr, nullptr, nullptr},
                                             noise, outputs};
                        for (int64_t i = 0; i < a.n; i++) {
                            const float *w = params + i * p.mlp.stride;
                            if (per_env) rollout_mlp_noisy_env<KIND, true>(a, i, T, last_obs, w, p);
                            else rollout_mlp_noisy_env<KIND, false>(a, i, T, last_obs, w, p);
                        }
                        return invalid ? -2 : 0;
                    });
}

}  // extern "C"
