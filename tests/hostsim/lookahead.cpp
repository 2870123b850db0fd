// lookahead.cpp -- kernel B's CartPole lookahead and the step it predicts, compiled for the CPU.
//
// TEST INFRASTRUCTURE (never shipped, never imported by gym_b200/): includes gym_b200/csrc/per_env.cuh through
// tests/hostsim/cuda_shim.h and evaluates, for caller-owned states, Env<CARTPOLE>::will_terminate against the
// `terminated` of Env<CARTPOLE>::step, and will_reset against advance_env's return.  tests/test_cartpole_lookahead_cpu.py
// checks that they agree bit for bit.
#include "cuda_shim.h"

#include <type_traits>

#include "../../gym_b200/csrc/rng.cuh"
#include "../../gym_b200/csrc/envs.cuh"
#include "../../gym_b200/csrc/box2d_consts.h"
#include "../../gym_b200/csrc/per_env.cuh"

namespace {

// a sink that drops advance_env's outputs
struct NullSink {
    template <int D, typename I> void obs(I, const float (&)[D]) const {}
    template <typename I> void scalars(I, double, uint8_t, uint8_t) const {}
    template <int S, typename I> void state(I, const double (&)[S]) const {}
    template <typename I> void elapsed(I, int32_t) const {}
    template <int D, typename I> void final_obs(I, const float (&)[D]) const {}
};

}  // namespace

extern "C" {

// n states [n][4] with their TimeLimit counters and actions: will_terminate and Env::step's `terminated`,
// will_reset and advance_env's return
void hs_cartpole_lookahead(const double *state_aos, const int32_t *elapsed, const int64_t *actions, int64_t n,
                           int32_t max_steps, int32_t autoreset, uint8_t *pred_term, uint8_t *step_term,
                           uint8_t *pred_reset, uint8_t *step_reset) {
    using E = bgym::Env<B200GYM_CARTPOLE>;
    unsigned long long invalid = 0, invalid_seen = 0;
    uint8_t flag = 0;
    StepArgs a{};
    a.invalid = &invalid;
    a.invalid_seen = &invalid_seen;
    a.flags = &flag;
    a.max_steps = max_steps;
    a.autoreset = autoreset;
    for (int64_t i = 0; i < n; i++) {
        double s[4], s2[4];
        for (int k = 0; k < 4; k++) s[k] = s2[k] = state_aos[4 * i + k];
        float obs[4];
        double reward;
        bool term;
        pred_term[i] = E::will_terminate(s);
        pred_reset[i] = will_reset<B200GYM_CARTPOLE>(a, s, elapsed[i], actions[i]);
        E::step(s, elapsed[i] == 0, actions[i] == 1 ? 1 : 0, 0.0f, 0.0, obs, reward, term);
        step_term[i] = term;
        flag = 0;
        step_reset[i] = advance_env<B200GYM_CARTPOLE>(a, NullSink{}, (int64_t)0, s2, elapsed[i], actions[i], 0.0f);
    }
}

}  // extern "C"
