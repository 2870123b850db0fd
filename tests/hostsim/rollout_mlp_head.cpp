// rollout_mlp_head.cpp -- the per-env drivers of rollout_mlp_head_kernel and rollout_mlp_noisy_head_kernel
// (rollout_mlp_head_env, rollout_mlp_noisy_head_env), compiled for the CPU.
//
// TEST INFRASTRUCTURE (never shipped, never imported by gym_b200/): includes gym_b200/csrc/per_env.cuh through
// rollout.cpp and drives the two drivers over the batch with plain loops, as the kernels do one env per thread.  The
// activation and the head are run-time codes here, dispatched to the same template instantiations the kernels use.
// mlp_tanh and head_exp are the host C library's tanhf and expf.  tests/test_rollout_mlp_head_cpu.py compares them
// with a numpy restatement that calls those same functions through ctypes.
#include "rollout.cpp"

namespace {

// fn(ACT, HEAD) as std::integral_constants for the run-time codes, -1 for any other code
template <typename Fn>
int64_t head_dispatch(int act, int head, Fn fn) {
    using R = std::integral_constant<int, B200GYM_MLP_RELU>;
    using Th = std::integral_constant<int, B200GYM_MLP_TANH>;
    using Ht = std::integral_constant<int, B200GYM_HEAD_TANH>;
    using Hn = std::integral_constant<int, B200GYM_HEAD_TANH_NORMAL>;
    if (act == B200GYM_MLP_RELU && head == B200GYM_HEAD_TANH) return fn(R{}, Ht{});
    if (act == B200GYM_MLP_RELU && head == B200GYM_HEAD_TANH_NORMAL) return fn(R{}, Hn{});
    if (act == B200GYM_MLP_TANH && head == B200GYM_HEAD_TANH) return fn(Th{}, Ht{});
    if (act == B200GYM_MLP_TANH && head == B200GYM_HEAD_TANH_NORMAL) return fn(Th{}, Hn{});
    return -1;
}

}  // namespace

extern "C" {

// T steps of rollout_mlp_head_env for every env of the batch (a classic Box kind): summary mode when returns is not
// null, and then the per-step pointers are ignored
int64_t hs_mlp_head_rollout(const Batch *B, const float *params, int per_env, int h1, int h2, int32_t T, int act,
                            int head, const float *bounds, void *actions_out, float *obs, double *reward,
                            uint8_t *term, uint8_t *trunc, float *final_obs, double *returns, int32_t *lengths,
                            uint8_t *ended, float *last_obs) {
    unsigned long long invalid = 0, seen = 0;
    const bool summary = returns != nullptr;
    const StepArgs a = summary ? args_of(*B, &invalid, &seen, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr)
                               : args_of(*B, &invalid, &seen, actions_out, obs, reward, term, trunc, final_obs);
    const HeadBounds hb{bounds[0], bounds[1], bounds[2], bounds[3]};
    return dispatch(B->kind, B200GYM_ACT_F32, [&](auto k, auto *) -> int64_t {
        constexpr int KIND = decltype(k)::value;
        if constexpr (bgym::Env<KIND>::A == 0) {
            return -1;
        } else {
            return head_dispatch(act, head, [&](auto ac, auto hd) -> int64_t {
                constexpr int ACT = decltype(ac)::value, HEAD = decltype(hd)::value;
                constexpr int K = head_outputs<HEAD>(bgym::Env<KIND>::A), D = bgym::Env<KIND>::D;
                const int64_t P = mlp_param_count<K, D>(h1, h2);
                const bool vec = h1 % 4 == 0 && (!per_env || P % 4 == 0);
                const MlpHeadArgs p{{params, per_env ? P : 0, h1, h2, vec ? 1 : 0, returns, lengths, ended}, nullptr,
                                    nullptr, hb};
                for (int64_t i = 0; i < a.n; i++) {
                    const float *w = params + i * p.mlp.stride;
                    if (per_env) {
                        if (summary) rollout_mlp_head_env<KIND, true, true, ACT, HEAD>(a, i, T, last_obs, w, p);
                        else rollout_mlp_head_env<KIND, false, true, ACT, HEAD>(a, i, T, last_obs, w, p);
                    } else {
                        if (summary) rollout_mlp_head_env<KIND, true, false, ACT, HEAD>(a, i, T, last_obs, w, p);
                        else rollout_mlp_head_env<KIND, false, false, ACT, HEAD>(a, i, T, last_obs, w, p);
                    }
                }
                return invalid ? -2 : 0;
            });
        }
    });
}

// T steps of rollout_mlp_noisy_head_env for every env of the batch (a classic Box kind)
int64_t hs_mlp_noisy_head_rollout(const Batch *B, const float *params, int per_env, int h1, int h2, int32_t T, int act,
                                  int head, const float *bounds, const float *noise, float *outputs, void *actions_out,
                                  float *obs, double *reward, uint8_t *term, uint8_t *trunc, float *final_obs,
                                  float *last_obs) {
    unsigned long long invalid = 0, seen = 0;
    const StepArgs a = args_of(*B, &invalid, &seen, actions_out, obs, reward, term, trunc, final_obs);
    const HeadBounds hb{bounds[0], bounds[1], bounds[2], bounds[3]};
    return dispatch(B->kind, B200GYM_ACT_F32, [&](auto k, auto *) -> int64_t {
        constexpr int KIND = decltype(k)::value;
        if constexpr (bgym::Env<KIND>::A == 0) {
            return -1;
        } else {
            return head_dispatch(act, head, [&](auto ac, auto hd) -> int64_t {
                constexpr int ACT = decltype(ac)::value, HEAD = decltype(hd)::value;
                constexpr int K = head_outputs<HEAD>(bgym::Env<KIND>::A), D = bgym::Env<KIND>::D;
                const int64_t P = mlp_param_count<K, D>(h1, h2);
                const bool vec = h1 % 4 == 0 && (!per_env || P % 4 == 0);
                const MlpHeadArgs p{{params, per_env ? P : 0, h1, h2, vec ? 1 : 0, nullptr, nullptr, nullptr}, noise,
                                    outputs, hb};
                for (int64_t i = 0; i < a.n; i++) {
                    const float *w = params + i * p.mlp.stride;
                    if (per_env) rollout_mlp_noisy_head_env<KIND, true, ACT, HEAD>(a, i, T, last_obs, w, p);
                    else rollout_mlp_noisy_head_env<KIND, false, ACT, HEAD>(a, i, T, last_obs, w, p);
                }
                return invalid ? -2 : 0;
            });
        }
    });
}

}  // extern "C"
