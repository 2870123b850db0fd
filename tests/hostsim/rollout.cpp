// rollout.cpp -- the per-env drivers of rollout_kernel and of kernel A, compiled for the CPU.
//
// TEST INFRASTRUCTURE (never shipped, never imported by gym_b200/): includes gym_b200/csrc/per_env.cuh through
// tests/hostsim/cuda_shim.h and runs, over caller-owned arrays of the handle's layout (state [S][n], elapsed [n],
// flags [n], PCG64 records [n][4]), reset_kernel's driver, kernel A's step (advance_env for every env, then reset_env
// for those whose episode ended) and rollout_env for every env.  tests/test_rollout_cpu.py checks that one rollout
// equals T steps bit for bit, for every classic kind, action dtype and TimeLimit / autoreset setting.  The argument
// set-up copies make_args and launch_rollout_kind.
#include "cuda_shim.h"

#include <type_traits>
#include <vector>

#include "../../gym_b200/csrc/rng.cuh"
#include "../../gym_b200/csrc/envs.cuh"
#include "../../gym_b200/csrc/box2d_consts.h"
#include "../../gym_b200/csrc/per_env.cuh"

namespace {

// the handle's per-env arrays and configuration (mirrored by rollout_sim.Batch)
struct Batch {
    int32_t kind, max_steps, autoreset, pad;
    int64_t n;
    double param0;
    double *state;
    int32_t *elapsed;
    uint8_t *flags;
    uint64_t *rng;
};

StepArgs args_of(const Batch &B, unsigned long long *invalid, unsigned long long *seen, const void *actions, float *obs,
                 double *reward, uint8_t *term, uint8_t *trunc, float *final_obs) {
    StepArgs a{};
    a.state = B.state; a.elapsed = B.elapsed; a.flags = B.flags; a.rng = B.rng;
    a.invalid = invalid; a.invalid_seen = seen;
    a.actions = actions; a.obs = obs; a.reward = reward; a.terminated = term; a.truncated = trunc;
    a.final_obs = final_obs;
    a.n = B.n; a.first = 0; a.count = B.n;
    a.max_steps = B.max_steps; a.autoreset = B.autoreset; a.param0 = B.param0;
    return a;
}

// fn(std::integral_constant<int, KIND>, (ActT *)nullptr) for the batch's kind and the action dtype code
template <typename Fn>
int64_t dispatch(int kind, int dtype, Fn fn) {
    auto typed = [&](auto k) -> int64_t {
        if constexpr (bgym::Env<decltype(k)::value>::A == 0) {
            switch (dtype) {
            case B200GYM_ACT_I64: return fn(k, (long long *)nullptr);
            case B200GYM_ACT_I32: return fn(k, (int *)nullptr);
            case B200GYM_ACT_U8: return fn(k, (unsigned char *)nullptr);
            default: return -1;
            }
        } else {
            return dtype == B200GYM_ACT_F32 ? fn(k, (float *)nullptr) : -1;
        }
    };
    switch (kind) {
    case B200GYM_CARTPOLE: return typed(std::integral_constant<int, B200GYM_CARTPOLE>{});
    case B200GYM_MOUNTAINCAR: return typed(std::integral_constant<int, B200GYM_MOUNTAINCAR>{});
    case B200GYM_MOUNTAINCAR_CONT: return typed(std::integral_constant<int, B200GYM_MOUNTAINCAR_CONT>{});
    case B200GYM_PENDULUM: return typed(std::integral_constant<int, B200GYM_PENDULUM>{});
    case B200GYM_ACROBOT: return typed(std::integral_constant<int, B200GYM_ACROBOT>{});
    }
    return -1;
}

}  // namespace

extern "C" {

// b200gym_seed_range: env i seeded with base + first + i
void hs_ro_seed_range(const Batch *B, const uint32_t base[4], int64_t first) {
    using bgym::u128;
    const u128 b = ((u128)base[3] << 96) | ((u128)base[2] << 64) | ((u128)base[1] << 32) | (u128)base[0];
    for (int64_t i = 0; i < B->n; i++) {
        const u128 seed = b + (u128)(uint64_t)(first + i);
        const uint32_t ent[4] = {(uint32_t)seed, (uint32_t)(seed >> 32), (uint32_t)(seed >> 64), (uint32_t)(seed >> 96)};
        bgym::Pcg64 g;
        bgym::pcg64_from_entropy(g, ent);
        bgym::pcg64_store_full(&B->rng[4 * i], g);
    }
}

// reset_kernel over every env; bounds NULL: the kind's defaults
int64_t hs_ro_reset(const Batch *B, const double *bounds, float *obs) {
    return dispatch(B->kind, B->kind == B200GYM_CARTPOLE || B->kind == B200GYM_MOUNTAINCAR || B->kind == B200GYM_ACROBOT
                                 ? B200GYM_ACT_I64 : B200GYM_ACT_F32,
                    [&](auto k, auto *) -> int64_t {
                        constexpr int KIND = decltype(k)::value;
                        double lo, hi;
                        bgym::Env<KIND>::default_bounds(lo, hi);
                        if (bounds) { lo = bounds[0]; hi = bounds[1]; }
                        for (int64_t i = 0; i < B->n; i++)
                            reset_env_bounded<KIND>(B->state, B->elapsed, B->flags, B->rng, obs, B->n, i, lo, hi);
                        return 0;
                    });
}

// one b200gym_step as kernel A runs it -> the number of invalid actions met (-1: bad kind / dtype)
int64_t hs_ro_step(const Batch *B, int dtype, const void *actions, float *obs, double *reward, uint8_t *term,
                   uint8_t *trunc, float *final_obs) {
    unsigned long long invalid = 0, seen = 0;
    const StepArgs a = args_of(*B, &invalid, &seen, actions, obs, reward, term, trunc, final_obs);
    const int64_t rc = dispatch(B->kind, dtype, [&](auto k, auto *tag) -> int64_t {
        constexpr int KIND = decltype(k)::value;
        using ActT = std::remove_pointer_t<decltype(tag)>;
        using E = bgym::Env<KIND>;
        const DirectSinkT<false> sink{a};
        std::vector<int64_t> resets;
        for (int64_t i = 0; i < a.n; i++) {
            double s[E::S];
            for (int k2 = 0; k2 < E::S; k2++) s[k2] = a.state[k2 * a.n + i];
            long long action_int = 0;
            float a0 = 0.0f;
            decode_action<KIND>(__ldg(reinterpret_cast<const ActT *>(a.actions) + i), action_int, a0);
            if (advance_env<KIND>(a, sink, i, s, a.elapsed[i], action_int, a0)) resets.push_back(i);
        }
        for (const int64_t i : resets) reset_env<KIND>(a, sink, i);
        return 0;
    });
    return rc < 0 ? rc : (int64_t)invalid;
}

// one b200gym_rollout of T steps as rollout_kernel runs it -> the number of invalid actions met (-1: bad kind / dtype)
int64_t hs_ro_rollout(const Batch *B, int dtype, int32_t T, const void *actions, float *obs, double *reward,
                      uint8_t *term, uint8_t *trunc, float *final_obs, float *last_obs) {
    unsigned long long invalid = 0, seen = 0;
    const StepArgs a = args_of(*B, &invalid, &seen, actions, obs, reward, term, trunc, final_obs);
    const int64_t rc = dispatch(B->kind, dtype, [&](auto k, auto *tag) -> int64_t {
        for (int64_t i = 0; i < a.n; i++)
            rollout_env<decltype(k)::value, std::remove_pointer_t<decltype(tag)>>(a, i, T, last_obs);
        return 0;
    });
    return rc < 0 ? rc : (int64_t)invalid;
}

}  // extern "C"
