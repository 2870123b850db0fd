// rollout_actor_critic.cpp -- the per-env drivers of rollout_actor_critic_kernel and gae_kernel, compiled for the CPU.
//
// TEST INFRASTRUCTURE (never shipped, never imported by gym_b200/): includes gym_b200/csrc/per_env.cuh through
// tests/hostsim/cuda_shim.h (by way of rollout.cpp, whose batch layout and reset / step entry points it shares) and runs
// rollout_actor_critic_env for every env, then gae_env for every env, as the two launches of
// b200gym_rollout_actor_critic do.  The actor and the critic are read where the kernel reads their shared-memory copies.
// tests/test_rollout_actor_critic_cpu.py compares one call with a numpy restatement of the actor plus the noise, the
// critic, T kernel-A steps of the same batch and the GAE recursion; hs_gae runs gae_env alone on hand-made inputs.
#include "rollout.cpp"

extern "C" {

// one b200gym_rollout_actor_critic call of T steps (h2 = 0: one hidden layer; act: a b200gym_mlp_activation), noise
// and outputs [T][n][K], values [T + 1][n], advantages [T][n] -> 0 (-1: bad kind)
int64_t hs_actor_critic_rollout(const Batch *B, const float *actor, const float *critic, int h1, int h2, int act,
                                int32_t T, const float *noise, float *outputs, void *actions_out, float *obs,
                                double *reward, uint8_t *term, uint8_t *trunc, float *final_obs, float *values,
                                float *advantages, float g, float gl, float *last_obs) {
    unsigned long long invalid = 0, seen = 0;
    const StepArgs a = args_of(*B, &invalid, &seen, actions_out, obs, reward, term, trunc, final_obs);
    const bool vec = h1 % 4 == 0;
    const ActorCriticArgs p{{{actor, 0, h1, h2, vec ? 1 : 0, nullptr, nullptr, nullptr}, noise, outputs}, critic, values,
                            advantages};
    const int64_t rc = dispatch(
        B->kind, B->kind == B200GYM_CARTPOLE || B->kind == B200GYM_MOUNTAINCAR || B->kind == B200GYM_ACROBOT
                     ? B200GYM_ACT_I64 : B200GYM_ACT_F32,
        [&](auto k, auto *) -> int64_t {
            constexpr int KIND = decltype(k)::value;
            for (int64_t i = 0; i < a.n; i++) {
                if (act == B200GYM_MLP_TANH)
                    rollout_actor_critic_env<KIND, B200GYM_MLP_TANH>(a, i, T, last_obs, actor, critic, p);
                else rollout_actor_critic_env<KIND, B200GYM_MLP_RELU>(a, i, T, last_obs, actor, critic, p);
            }
            return invalid ? -2 : 0;
        });
    if (rc) return rc;
    for (int64_t i = 0; i < a.n; i++) gae_env(i, a.n, T, g, gl, reward, term, trunc, values, advantages);
    return 0;
}

// gae_kernel's per-env work for every env of [T][n] rows (values [T + 1][n]; adv holds V(final obs) where a step
// truncated without terminating)
void hs_gae(int64_t n, int32_t T, float g, float gl, const double *reward, const uint8_t *term, const uint8_t *trunc,
            const float *values, float *adv) {
    for (int64_t i = 0; i < n; i++) gae_env(i, n, T, g, gl, reward, term, trunc, values, adv);
}

}  // extern "C"
