// rollout_policy_norm.cpp -- the per-env drivers of rollout_linear_norm_kernel and rollout_mlp_norm_kernel, compiled
// for the CPU.
//
// TEST INFRASTRUCTURE (never shipped, never imported by gym_b200/): includes gym_b200/csrc/per_env.cuh through
// tests/hostsim/cuda_shim.h (by way of rollout.cpp, whose batch layout and reset / step entry points it shares).  The
// statistics are staged as the kernels stage them, mean[D] and sd[D] = norm_sd(var[D], eps), once per call (mean null:
// raw inputs); a shared MLP is read where the kernel reads its shared-memory copy.  tests/test_rollout_policy_norm_cpu.py
// compares the drivers with a numpy restatement and with the drivers without normalisation.
#include "rollout.cpp"

namespace {

template <typename F>
int64_t policy_norm_dispatch(const Batch *B, const double *mean, const double *var, double eps, double *sd, F f) {
    return dispatch(B->kind, B->kind == B200GYM_CARTPOLE || B->kind == B200GYM_MOUNTAINCAR || B->kind == B200GYM_ACROBOT
                                 ? B200GYM_ACT_I64 : B200GYM_ACT_F32,
                    [&](auto k, auto *) -> int64_t {
                        constexpr int KIND = decltype(k)::value;
                        if (mean)
                            for (int c = 0; c < bgym::Env<KIND>::D; c++) sd[c] = norm_sd(var[c], eps);
                        return f(k);
                    });
}

}  // namespace

extern "C" {

// one b200gym_rollout_linear_norm launch of T steps of a classic kind; returns NULL: per-step outputs, else the summary
// (actions ... final_obs unused) with the moments when sum is not null; mean NULL: raw inputs -> 0 (-1: bad kind)
int64_t hs_linear_norm_rollout(const Batch *B, const float *weight, const float *bias, int per_env, int32_t T,
                               void *actions_out, float *obs, double *reward, uint8_t *term, uint8_t *trunc,
                               float *final_obs, double *returns, int32_t *lengths, uint8_t *ended, float *last_obs,
                               const double *mean, const double *var, double eps, float clip, double *sum,
                               double *sumsq) {
    unsigned long long invalid = 0, seen = 0;
    const bool summary = returns != nullptr;
    const StepArgs a = summary ? args_of(*B, &invalid, &seen, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr)
                               : args_of(*B, &invalid, &seen, actions_out, obs, reward, term, trunc, final_obs);
    const ObsMomentArgs m{sum, sumsq};
    double sd[24];
    return policy_norm_dispatch(B, mean, var, eps, sd, [&](auto k) -> int64_t {
        constexpr int KIND = decltype(k)::value;
        const int64_t K = linear_logit_count<KIND>(), D = bgym::Env<KIND>::D;
        const LinearPolicyArgs p{weight, bias, per_env ? K * D : 0, per_env ? K : 0, returns, lengths, ended};
        for (int64_t i = 0; i < a.n; i++) {
            if (summary) rollout_linear_norm_env<KIND, true>(a, i, T, last_obs, p, mean, sd, clip, m);
            else rollout_linear_norm_env<KIND, false>(a, i, T, last_obs, p, mean, sd, clip, m);
        }
        return invalid ? -2 : 0;
    });
}

// one b200gym_rollout_mlp_norm launch (h2 = 0: one hidden layer; act: a b200gym_mlp_activation); the rest as
// hs_linear_norm_rollout
int64_t hs_mlp_norm_rollout(const Batch *B, const float *params, int per_env, int h1, int h2, int act, int32_t T,
                            void *actions_out, float *obs, double *reward, uint8_t *term, uint8_t *trunc,
                            float *final_obs, double *returns, int32_t *lengths, uint8_t *ended, float *last_obs,
                            const double *mean, const double *var, double eps, float clip, double *sum,
                            double *sumsq) {
    unsigned long long invalid = 0, seen = 0;
    const bool summary = returns != nullptr;
    const StepArgs a = summary ? args_of(*B, &invalid, &seen, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr)
                               : args_of(*B, &invalid, &seen, actions_out, obs, reward, term, trunc, final_obs);
    const ObsMomentArgs m{sum, sumsq};
    double sd[24];
    return policy_norm_dispatch(B, mean, var, eps, sd, [&](auto k) -> int64_t {
        constexpr int KIND = decltype(k)::value, R = B200GYM_MLP_RELU, H = B200GYM_MLP_TANH;
        constexpr int K = linear_logit_count<KIND>(), D = bgym::Env<KIND>::D;
        const int64_t P = mlp_param_count<K, D>(h1, h2);
        const bool vec = h1 % 4 == 0 && (!per_env || P % 4 == 0);
        const MlpPolicyArgs p{params, per_env ? P : 0, h1, h2, vec ? 1 : 0, returns, lengths, ended};
        for (int64_t i = 0; i < a.n; i++) {
            const float *w = params + i * p.stride;
            if (per_env) {
                if (summary) {
                    if (act == H) rollout_mlp_norm_env<KIND, true, true, H>(a, i, T, last_obs, w, p, mean, sd, clip, m);
                    else rollout_mlp_norm_env<KIND, true, true, R>(a, i, T, last_obs, w, p, mean, sd, clip, m);
                } else {
                    if (act == H) rollout_mlp_norm_env<KIND, false, true, H>(a, i, T, last_obs, w, p, mean, sd, clip, m);
                    else rollout_mlp_norm_env<KIND, false, true, R>(a, i, T, last_obs, w, p, mean, sd, clip, m);
                }
            } else {
                if (summary) {
                    if (act == H) rollout_mlp_norm_env<KIND, true, false, H>(a, i, T, last_obs, w, p, mean, sd, clip, m);
                    else rollout_mlp_norm_env<KIND, true, false, R>(a, i, T, last_obs, w, p, mean, sd, clip, m);
                } else {
                    if (act == H)
                        rollout_mlp_norm_env<KIND, false, false, H>(a, i, T, last_obs, w, p, mean, sd, clip, m);
                    else rollout_mlp_norm_env<KIND, false, false, R>(a, i, T, last_obs, w, p, mean, sd, clip, m);
                }
            }
        }
        return invalid ? -2 : 0;
    });
}

}  // extern "C"
