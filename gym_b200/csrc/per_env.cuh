// per_env.cuh -- the per-env drivers of the step and reset kernels: everything one thread does for the env it owns,
// between "this thread owns env i" and the env's dynamics.  It reads the env's inputs, decodes the action, calls the
// dynamics (envs.cuh, lunar.cuh, walker.cuh), applies TimeLimit and the same-step autoreset, and writes the outputs.
//
// The kernels in b200gym.cu keep their thread and warp logic (indices, tiles, shared-memory lists, warp ballots,
// grid-stride loops) and call these functions for the per-env part.  tests/hostsim/hostsim.cpp compiles this header
// with g++ and drives the same functions with plain loops, in the order the kernels are launched, so that the CPU
// suite runs the code the kernels run.
#pragma once

#include <cstdint>
#include <type_traits>

#include "../../include/b200gym.h"
#include "envs.cuh"
#include "lunar.cuh"
#include "rng.cuh"
#include "walker.cuh"

struct StepArgs {
    double *state;
    int32_t *elapsed;
    uint8_t *flags;
    uint64_t *rng;
    unsigned long long *invalid;
    unsigned long long *invalid_seen;   // device-mapped host word, see b200gym_invalid_seen
    uint32_t *lunar_rec;
    const void *actions;
    float *obs;
    double *reward;
    uint8_t *terminated;
    uint8_t *truncated;
    float *final_obs;
    int64_t n;        // envs in the handle (SoA stride)
    int64_t first;    // sub-range processed by this launch
    int64_t count;
    int32_t max_steps;
    int32_t autoreset;
    double param0;
    lunar::Opts lunar_opts;   // LunarLander constructor variants (uniform over the batch)
    // Box2D tasks: envs whose episode ended in this launch are appended here (offset from `first`) and reset by
    // the *_reset_list_kernel that follows on the stream; nullptr: reset inline
    int32_t *reset_list;
    int32_t *reset_count;
    // Box2D tasks: envs whose step may contain a continuous-collision event (b2l::toi_needed) are parked after the
    // discrete solve -- world record + the sweep starts / env intermediates in toi_mid -- and finished by the
    // *_toi_kernel that follows on the stream, in warps full of such envs; nullptr: everything inline
    int32_t *toi_list;
    int32_t *toi_count;
    uint32_t *toi_mid;
    // fused all-gather: the step barrier in kernel G's tail (null = the separate p2p_sync_kernel / no exchange).  The
    // last CTA of the launch to finish its pushes publishes "my rows of step `p2p_step` are in your buffers" to every
    // peer and waits for theirs, so the exchange costs no launch of its own
    unsigned int *p2p_done;                       // device counter of finished CTAs (reset by the last one)
    unsigned long long *const *p2p_peer_flags;    // [world] -> rank r's flag words (mapped)
    const unsigned long long *p2p_my_flags;
    int *p2p_timed_out;
    unsigned long long p2p_step, p2p_timeout_ns;
    int32_t p2p_world, p2p_rank;
    int32_t bulk_sink;   // 1: use kernel G's staged bulk stores even without peers (host path: the output arrays are
                         // mapped host memory, where many small stores are what hurts)
    // fused all-gather (multi-GPU): every result is ALSO stored into the same rows of the peers'
    // gather buffers over NVLink (peer-mapped pointers, slice offset already applied)
    int32_t npeer;
    float *peer_obs[B200GYM_MAX_PEERS];
    double *peer_reward[B200GYM_MAX_PEERS];
    uint8_t *peer_term[B200GYM_MAX_PEERS];
    uint8_t *peer_trunc[B200GYM_MAX_PEERS];
};

template <int D, typename I>
__device__ __forceinline__ void store_row(float *base, I i, const float (&v)[D]) {
    if constexpr (D == 4) {
        reinterpret_cast<float4 *>(base)[i] = make_float4(v[0], v[1], v[2], v[3]);
    } else if constexpr (D == 2) {
        reinterpret_cast<float2 *>(base)[i] = make_float2(v[0], v[1]);
    } else if constexpr (D == 8 || D == 24) {
        float4 *p = reinterpret_cast<float4 *>(base) + (D / 4) * i;
#pragma unroll
        for (int k = 0; k < D / 4; k++) p[k] = make_float4(v[4 * k], v[4 * k + 1], v[4 * k + 2], v[4 * k + 3]);
    } else if constexpr (D == 6) {
        float2 *p = reinterpret_cast<float2 *>(base) + 3 * i;
        p[0] = make_float2(v[0], v[1]);
        p[1] = make_float2(v[2], v[3]);
        p[2] = make_float2(v[4], v[5]);
    } else {
#pragma unroll
        for (int k = 0; k < D; k++) base[i * D + k] = v[k];
    }
}

template <int D, typename I>
__device__ __forceinline__ void store_obs_all(const StepArgs &a, I i, const float (&v)[D]) {
    store_row<D>(a.obs, i, v);
    for (int p = 0; p < a.npeer; p++) store_row<D>(a.peer_obs[p], i, v);
}

template <typename I>
__device__ __forceinline__ void store_scalars_all(const StepArgs &a, I i, double reward, uint8_t term,
                                                  uint8_t trunc) {
    a.reward[i] = reward;
    a.terminated[i] = term;
    a.truncated[i] = trunc;
    for (int p = 0; p < a.npeer; p++) {
        a.peer_reward[p][i] = reward;
        a.peer_term[p][i] = term;
        a.peer_trunc[p][i] = trunc;
    }
}

// Where the results of env i go.  DirectSink: straight to the caller's arrays (and, when peers are mapped,
// to theirs) with per-thread stores; final_obs rows (info["final_observation"]) are never peer-mapped.  The kernels that stage their outputs in shared memory have sinks of their own
// (b200gym.cu: StagedSink, InPlaceSink).
// PEERS = false: the caller knows there are no peer-mapped destinations (single-GPU step), so the per-destination
// loops and their constant-bank traffic disappear from the hot loop.
template <bool PEERS>
struct DirectSinkT {
    const StepArgs &a;
    template <int D, typename I>
    __device__ __forceinline__ void obs(I i, const float (&v)[D]) const {
        if constexpr (PEERS) store_obs_all<D>(a, i, v);
        else store_row<D>(a.obs, i, v);
    }
    template <typename I>
    __device__ __forceinline__ void scalars(I i, double reward, uint8_t term, uint8_t trunc) const {
        if constexpr (PEERS) store_scalars_all(a, i, reward, term, trunc);
        else { a.reward[i] = reward; a.terminated[i] = term; a.truncated[i] = trunc; }
    }
    template <int S, typename I>
    __device__ __forceinline__ void state(I i, const double (&s)[S]) const {
#pragma unroll
        for (int k = 0; k < S; k++) a.state[k * a.n + i] = s[k];
    }
    template <typename I>
    __device__ __forceinline__ void elapsed(I i, int32_t e) const { a.elapsed[i] = e; }
    template <int D, typename I>
    __device__ __forceinline__ void final_obs(I i, const float (&v)[D]) const {
        if (a.final_obs) store_row<D>(a.final_obs, i, v);
    }
};
using DirectSink = DirectSinkT<true>;

// ---- classic control -------------------------------------------------------------------------------------------

// The action of env i as advance_env takes it: an integer for a Discrete space, a float for Box(1)
template <int KIND, typename ActT>
__device__ __forceinline__ void decode_action(ActT av, long long &action_int, float &a0) {
    if constexpr (bgym::Env<KIND>::A == 0) action_int = (long long)av;
    else a0 = (float)av;
}

// Phase 1, by the thread that owns env i (its inputs are in registers): Env.step, TimeLimit,
// stores of reward / flags / final_obs, and -- unless the episode ended -- of the new state and
// observation.  Returns true when the env must be reset by phase 2.
template <int KIND, typename Sink, typename I>
__device__ __forceinline__ bool advance_env(const StepArgs &a, const Sink &sink, I i, double (&s)[bgym::Env<KIND>::S],
                                            int32_t elapsed, long long action_int, float a0) {
    using E = bgym::Env<KIND>;
    int act = 0;
    if constexpr (E::A == 0) {
        if (action_int < 0 || action_int >= E::NACT) {
            // the reference raises (cartpole.py:132 / mountain_car.py:128-130 / acrobot.py:199): leave the env
            // untouched, count it (sticky), return a NaN reward and the env's CURRENT observation, so that the
            // double-buffered output row does not show the observation of two steps ago
            atomicAdd(a.invalid, 1ULL);
            *reinterpret_cast<volatile unsigned long long *>(a.invalid_seen) = 1ULL;
            float cur[E::D];
            E::observe(s, cur);
            sink.scalars(i, __longlong_as_double(0x7ff8000000000000LL), 0, 0);
            sink.template obs<E::D>(i, cur);
            return false;
        }
        act = (int)action_int;
    }

    float obs[E::D];
    double reward;
    bool terminated;
    E::step(s, elapsed == 0, act, a0, a.param0, obs, reward, terminated);

    if (!a.autoreset) {
        if constexpr (KIND == B200GYM_CARTPOLE) {
            // cartpole.py:169-184: reward 0.0 once the pole has already fallen
            const uint8_t f = a.flags[i];
            if (terminated) {
                if (f & 1) reward = 0.0;
                else a.flags[i] = f | 1;
            }
        }
    }

    elapsed += 1;                                                        // time_limit.py:51
    const bool truncated = (a.max_steps > 0) && (elapsed >= a.max_steps);  // :53-54
    const bool needs_reset = (terminated || truncated) && a.autoreset;   // sync_vector_env.py:152-156

    sink.scalars(i, reward, terminated ? 1 : 0, truncated ? 1 : 0);
    if (needs_reset) {
        sink.template final_obs<E::D>(i, obs);                            // info["final_observation"]
    } else {
        sink.template state<E::S>(i, s);
        sink.elapsed(i, elapsed);
        sink.template obs<E::D>(i, obs);
    }
    return needs_reset;
}

// Whether advance_env will return true for these inputs, known before it runs: kernel B uses it to fetch the PCG64
// records of a tile's finishing envs early.  Only CartPole's termination can be seen ahead (Env::will_terminate); the
// other kinds answer false.  A kernel must not depend on the answer for correctness
template <int KIND>
__device__ __forceinline__ bool will_reset(const StepArgs &a, const double (&s)[bgym::Env<KIND>::S], int32_t elapsed,
                                           long long action_int) {
    using E = bgym::Env<KIND>;
    if constexpr (KIND == B200GYM_CARTPOLE) {
        if (!a.autoreset || action_int < 0 || action_int >= E::NACT) return false;
        return ((a.max_steps > 0) && (elapsed + 1 >= a.max_steps)) || E::will_terminate(s);
    } else {
        return false;
    }
}

// Phase 2: the unseeded env.reset() of the autoreset (sync_vector_env.py:154) for env i, by
// whichever thread picked it off the CTA's compacted list.  reset_env_from: the same with env i's PCG64 record
// loaded and written back by the caller
template <int KIND, typename Sink, typename I>
__device__ __forceinline__ void reset_env_from(const Sink &sink, I i, bgym::Pcg64 &g) {
    using E = bgym::Env<KIND>;
    double s[E::S];
    float obs[E::D];
    double lo, hi;
    E::default_bounds(lo, hi);
    E::reset(s, g, lo, hi, obs);
    sink.template state<E::S>(i, s);
    sink.elapsed(i, 0);                                                  // time_limit.py:67
    sink.template obs<E::D>(i, obs);
}

template <int KIND, typename Sink, typename I>
__device__ __forceinline__ void reset_env(const StepArgs &a, const Sink &sink, I i) {
    bgym::Pcg64 g = bgym::pcg64_load(a.rng + 4 * (size_t)i);
    reset_env_from<KIND>(sink, i, g);
    bgym::pcg64_store(a.rng + 4 * (size_t)i, g);
}

// ---- rollouts (b200gym_rollout) ---------------------------------------------------------------------------------

// A store the rollout's outputs make once and never read back: evict-first on the device, where T steps of outputs
// are far larger than L2; a plain store in the host build
template <typename T>
__device__ __forceinline__ void store_once(T *p, T v) {
#ifdef __CUDA_ARCH__
    __stcs(p, v);
#else
    *p = v;
#endif
}

// The sink of one rollout step: the state and TimeLimit counter go to the thread's registers, the outputs to the rows
// of slice t (the pointers are advanced by one slice per step), and on the last step the observation also to `last`,
// the handle's own observation buffer
template <int KIND>
struct RolloutSink {
    double (&s)[bgym::Env<KIND>::S];
    int32_t &el;
    float *o;
    double *r;
    uint8_t *te, *tr;
    float *fin;    // null: no final observations
    float *last;   // null but on the last step
    template <int D, typename I>
    __device__ __forceinline__ void obs_row(float *base, I i, const float (&v)[D]) const {
        if constexpr (D == 4) {
            store_once(reinterpret_cast<float4 *>(base) + i, make_float4(v[0], v[1], v[2], v[3]));
        } else if constexpr (D == 2) {
            store_once(reinterpret_cast<float2 *>(base) + i, make_float2(v[0], v[1]));
        } else {
#pragma unroll
            for (int k = 0; k < D; k++) store_once(base + i * D + k, v[k]);
        }
    }
    template <int D, typename I>
    __device__ __forceinline__ void obs(I i, const float (&v)[D]) const {
        obs_row<D>(o, i, v);
        if (last) store_row<D>(last, i, v);
    }
    template <typename I>
    __device__ __forceinline__ void scalars(I i, double reward, uint8_t term, uint8_t trunc) const {
        store_once(r + i, reward);
        store_once(te + i, term);
        store_once(tr + i, trunc);
    }
    template <int S, typename I>
    __device__ __forceinline__ void state(I, const double (&v)[S]) const {
#pragma unroll
        for (int k = 0; k < S; k++) s[k] = v[k];
    }
    template <typename I>
    __device__ __forceinline__ void elapsed(I, int32_t e) const { el = e; }
    template <int D, typename I>
    __device__ __forceinline__ void final_obs(I i, const float (&v)[D]) const {
        if (fin) obs_row<D>(fin, i, v);
    }
    // on to the rows of the next slice
    __device__ __forceinline__ void next(int64_t n) {
        o += n * bgym::Env<KIND>::D;
        r += n;
        te += n;
        tr += n;
        if (fin) fin += n * bgym::Env<KIND>::D;
    }
};

// Where a rollout's actions come from.  Row t of the [T][n] array at a.actions holds the actions of step t; the
// driver walks it with one pointer, `row`.  ReadActions: the caller wrote it (b200gym_rollout), so env i's action is
// read from it
struct ReadActions {
    template <typename ActT>
    __device__ __forceinline__ ActT action(const ActT *row, int64_t i) const { return __ldg(row + i); }
    __device__ __forceinline__ void next() const {}
};

// DrawActions: the rollout fills it (b200gym_rollout_sampled), drawing from the batched action space's stream.  Every
// classic kind has one action element per env (Discrete, or Box of shape (1,)), so env i's action of step t is draw
// t * n + i: g starts before draw i, takes one draw per step and then hops the n - 1 draws of the other envs
// (state -> hop_mult * state + hop_plus).  The value drawn is stored to the row and decoded like a value read from it
struct DrawActions {
    bgym::Pcg64 g;
    bgym::u128 hop_mult, hop_plus;
    double p0, p1;   // Discrete: n_choices (p1 unused); Box(1): low, high
    template <typename ActT>
    __device__ __forceinline__ ActT action(const ActT *row, int64_t i) {
        ActT v;
        if constexpr (std::is_same<ActT, long long>::value) v = bgym::sample_multidiscrete(g, p0);
        else v = bgym::sample_box(g, p0, p1);
        store_once(const_cast<ActT *>(row) + i, v);
        return v;
    }
    __device__ __forceinline__ void next() { g.state = hop_mult * g.state + hop_plus; }
};

// T steps of env i (rollout_kernel, rollout_sampled_kernel), the same as T launches of kernel A: advance_env and,
// when the episode ended, reset_env, with the state and TimeLimit counter loaded once and stored once; the actions
// come from `src`.  a.actions, a.obs, a.reward, a.terminated, a.truncated and a.final_obs hold slice 0 of [T][n]
// arrays; CartPole's autoreset=False flag byte stays in global memory, where advance_env keeps it
template <int KIND, typename ActT, typename Src = ReadActions>
__device__ __forceinline__ void rollout_env(const StepArgs &a, int64_t i, int32_t T, float *last_obs,
                                            Src src = Src{}) {
    using E = bgym::Env<KIND>;
    const int64_t n = a.n;
    double s[E::S];
#pragma unroll
    for (int k = 0; k < E::S; k++) s[k] = a.state[k * n + i];
    int32_t elapsed = a.elapsed[i];
    const ActT *act = reinterpret_cast<const ActT *>(a.actions);
    RolloutSink<KIND> sink{s, elapsed, a.obs, a.reward, a.terminated, a.truncated, a.final_obs, nullptr};
    for (int32_t t = 0; t < T; t++) {
        if (t == T - 1) sink.last = last_obs;
        long long action_int = 0;
        float a0 = 0.0f;
        decode_action<KIND>(src.action(act, i), action_int, a0);
        if (advance_env<KIND>(a, sink, i, s, elapsed, action_int, a0)) reset_env<KIND>(a, sink, i);
        src.next();
        act += n;
        sink.o += n * E::D;
        sink.r += n;
        sink.te += n;
        sink.tr += n;
        if (sink.fin) sink.fin += n * E::D;
    }
#pragma unroll
    for (int k = 0; k < E::S; k++) a.state[k * n + i] = s[k];
    a.elapsed[i] = elapsed;
}

// What every thread of a rollout_sampled_kernel launch shares: the map of n - 1 draws (independent of inc, like
// SampleArgs.hop_geo, so that a graph replayed after a reseed cannot hold a stale hop) and the plan of the single
// action space
struct RolloutDraws {
    bgym::u128 hop_mult, hop_geo;
    double p0, p1;      // as DrawActions
    int jump_digits;    // hex digits of n - 1: the rows of kLcgJump the first jumps use
};

// ... with the actions drawn from `start`, the generator before draw 0 of the launch, into a.actions: a table jump
// to draw i, then DrawActions
template <int KIND>
__device__ __forceinline__ void rollout_sampled_env(const StepArgs &a, int64_t i, int32_t T, float *last_obs,
                                                    const RolloutDraws &d, const bgym::Pcg64 &start,
                                                    const bgym::LcgJumpTable &table) {
    using ActT = typename std::conditional<bgym::Env<KIND>::A == 0, long long, float>::type;
    DrawActions src{start, d.hop_mult, d.hop_geo * start.inc, d.p0, d.p1};
    bgym::pcg64_jump_table(src.g, (uint64_t)i, table);
    rollout_env<KIND, ActT>(a, i, T, last_obs, src);
}

// ---- closed-loop rollouts of a linear policy (b200gym_rollout_linear) ---------------------------------------------

// The logits z of the linear policy (weight (K, D) row-major, bias (K,)) at the float32 observation o: z[j] starts at
// bias[j] and adds weight[j, k] * o[k] for k = 0 .. D-1 in that order, every product and every sum rounded to float32
// (the library is built with -fmad=false and the host build with -ffp-contract=off, so nothing is fused)
template <int K, int D>
__device__ __forceinline__ void linear_logits(const float *w, const float *b, const float (&o)[D], float (&z)[K]) {
#pragma unroll
    for (int j = 0; j < K; j++) {
        float v = b[j];
#pragma unroll
        for (int k = 0; k < D; k++) v = v + w[j * D + k] * o[k];
        z[j] = v;
    }
}

// np.argmax(z): the index of the first NaN if any logit is NaN, otherwise of the first maximum
template <int K>
__device__ __forceinline__ int argmax_first(const float (&z)[K]) {
    float m = z[0];
    int best = 0;
#pragma unroll
    for (int j = 1; j < K; j++) {
        if (m == m && (z[j] != z[j] || z[j] > m)) {
            m = z[j];
            best = j;
        }
    }
    return best;
}

// The number of logits of a linear policy of kind KIND: the Discrete kinds' choices, the Box kinds' act_dim
template <int KIND>
constexpr int linear_logit_count() {
    return bgym::Env<KIND>::A == 0 ? bgym::Env<KIND>::NACT : bgym::Env<KIND>::A;
}

// LinearActions: the rollout computes them (b200gym_rollout_linear) from `o`, the observation the env last returned,
// which LinearSink keeps current: argmax_first of the logits for a Discrete kind, the logits themselves for a Box kind.
// The action is stored to the row unless SUMMARY (no per-step outputs) and decoded like a value read from it
template <int KIND, bool SUMMARY>
struct LinearActions {
    static constexpr int K = linear_logit_count<KIND>(), D = bgym::Env<KIND>::D;
    float w[K * D], b[K];
    const float (&o)[D];
    template <typename ActT>
    __device__ __forceinline__ ActT action(const ActT *row, int64_t i) const {
        float z[K];
        linear_logits<K, D>(w, b, o, z);
        ActT v;
        if constexpr (bgym::Env<KIND>::A == 0) v = (ActT)argmax_first<K>(z);
        else v = z[0];
        if constexpr (!SUMMARY) store_once(const_cast<ActT *>(row) + i, v);
        return v;
    }
};

// The sink of a linear-policy rollout: RolloutSink's, plus every observation the step produces (the step's own, or the
// reset observation after an autoreset) copied to `seen`, the policy's input of the next step.  SUMMARY: nothing is
// stored per step but the last observation; the reward and flags are folded into the episode summary in registers
template <int KIND, bool SUMMARY>
struct LinearSink : RolloutSink<KIND> {
    using Base = RolloutSink<KIND>;
    float (&seen)[bgym::Env<KIND>::D];
    double &ret;     // 0.0 + the rewards up to the first episode end, in step order
    int32_t &len;    // steps up to and including the first episode end
    bool &ended;
    template <int D, typename I>
    __device__ __forceinline__ void obs(I i, const float (&v)[D]) const {
        if constexpr (SUMMARY) {
            if (this->last) store_row<D>(this->last, i, v);
        } else {
            Base::template obs<D>(i, v);
        }
#pragma unroll
        for (int k = 0; k < D; k++) seen[k] = v[k];
    }
    template <typename I>
    __device__ __forceinline__ void scalars(I i, double reward, uint8_t term, uint8_t trunc) const {
        if constexpr (SUMMARY) {
            if (!ended) {
                ret = ret + reward;
                len += 1;
                ended = (term | trunc) != 0;
            }
        } else {
            Base::scalars(i, reward, term, trunc);
        }
    }
    template <int D, typename I>
    __device__ __forceinline__ void final_obs(I i, const float (&v)[D]) const {
        if constexpr (!SUMMARY) Base::template final_obs<D>(i, v);
    }
    __device__ __forceinline__ void next(int64_t n) {
        if constexpr (!SUMMARY) Base::next(n);
    }
};

// The parameters and summary outputs of a b200gym_rollout_linear launch.  Env i's policy is weight + i * w_stride
// (K * D floats) and bias + i * b_stride (K floats); strides 0: one policy shared by every env
struct LinearPolicyArgs {
    const float *weight, *bias;
    int64_t w_stride, b_stride;
    double *returns;    // [n], SUMMARY only
    int32_t *lengths;
    uint8_t *ended;
};

// T steps of env i under its linear policy (rollout_linear_kernel): rollout_env's loop with LinearActions and
// LinearSink.  (Routing rollout_env itself through one loop shared with this driver changes the code the compiler
// makes for the Pendulum and Acrobot rollout kernels, so the loop is kept twice.)  Step 0's input is observe() of the
// state just loaded: for the classic kinds the observation the env last returned is that function of its state, and
// the state, unlike the double-buffered observation rows, is where a CUDA graph replay finds the current one.  The
// parameters are loaded once.  SUMMARY: no per-step outputs, the episode summary stored once at the end
template <int KIND, bool SUMMARY>
__device__ __forceinline__ void rollout_linear_env(const StepArgs &a, int64_t i, int32_t T, float *last_obs,
                                                   const LinearPolicyArgs &p) {
    using E = bgym::Env<KIND>;
    using ActT = typename std::conditional<E::A == 0, long long, float>::type;
    using Src = LinearActions<KIND, SUMMARY>;
    const int64_t n = a.n;
    double s[E::S];
#pragma unroll
    for (int k = 0; k < E::S; k++) s[k] = a.state[k * n + i];
    int32_t elapsed = a.elapsed[i];
    float o[E::D];
    E::observe(s, o);
    Src src{{}, {}, o};
    const float *w = p.weight + i * p.w_stride, *b = p.bias + i * p.b_stride;
#pragma unroll
    for (int k = 0; k < Src::K * E::D; k++) src.w[k] = __ldg(w + k);
#pragma unroll
    for (int j = 0; j < Src::K; j++) src.b[j] = __ldg(b + j);
    double ret = 0.0;
    int32_t len = 0;
    bool ended = false;
    LinearSink<KIND, SUMMARY> sink{{s, elapsed, a.obs, a.reward, a.terminated, a.truncated, a.final_obs, nullptr},
                                   o, ret, len, ended};
    const ActT *act = reinterpret_cast<const ActT *>(a.actions);
    for (int32_t t = 0; t < T; t++) {
        if (t == T - 1) sink.last = last_obs;
        long long action_int = 0;
        float a0 = 0.0f;
        decode_action<KIND>(src.action(act, i), action_int, a0);
        if (advance_env<KIND>(a, sink, i, s, elapsed, action_int, a0)) reset_env<KIND>(a, sink, i);
        act += n;
        sink.next(n);
    }
#pragma unroll
    for (int k = 0; k < E::S; k++) a.state[k * n + i] = s[k];
    a.elapsed[i] = elapsed;
    if constexpr (SUMMARY) {
        p.returns[i] = ret;
        p.lengths[i] = len;
        p.ended[i] = ended ? 1 : 0;
    }
}

// ---- closed-loop rollouts of an MLP policy (b200gym_rollout_mlp) --------------------------------------------------

constexpr int kMlpMaxWidth = 64;   // the widest hidden layer b200gym_rollout_mlp takes

// The hidden layers' activation: z if z > 0 or z is NaN, else +0.0 (so NaN propagates and -0.0 becomes +0.0)
__device__ __forceinline__ float mlp_relu(float z) { return (z > 0.0f || z != z) ? z : 0.0f; }

// The tanh activation: CUDA's tanhf on the device, which compiles to the instruction sequence of torch.tanh's float32
// CUDA kernel (DESIGN.md §4.15), and the C library's tanhf in the host build.  b200gym_selftest_tanh evaluates it
__host__ __device__ __forceinline__ float mlp_tanh(float z) { return tanhf(z); }

// The activation ACT (B200GYM_MLP_RELU or B200GYM_MLP_TANH) of a hidden unit, chosen at compile time
template <int ACT>
__device__ __forceinline__ float mlp_act(float z) {
    static_assert(ACT == B200GYM_MLP_RELU || ACT == B200GYM_MLP_TANH, "unknown MLP activation");
    if constexpr (ACT == B200GYM_MLP_TANH) return mlp_tanh(z);
    else return mlp_relu(z);
}

// A parameter of the MLP: from device memory through the read-only path (GLOBAL, each env's own row), or from the
// CTA's shared copy
template <bool GLOBAL>
__device__ __forceinline__ float mlp_ld(const float *p) {
    if constexpr (GLOBAL) return __ldg(p);
    else return *p;
}
template <bool GLOBAL>
__device__ __forceinline__ float4 mlp_ld4(const float *p) {
    if constexpr (GLOBAL) return __ldg(reinterpret_cast<const float4 *>(p));
    else return *reinterpret_cast<const float4 *>(p);
}

// The K outputs z of the MLP D -> h1 (-> h2) -> K (h2 = 0: one hidden layer) whose packed parameters start at w: layer
// by layer the weight (out, in) row-major, then the bias (out,).  Every unit starts at its bias and adds
// weight[j, k] * x[k] for k = 0 .. in-1 in that order, every product and sum rounded to float32 (the library is built
// with -fmad=false and the host build with -ffp-contract=off), as linear_logits; a hidden unit then goes through
// mlp_act<ACT>.  The first hidden layer is held in a register array of kMlpMaxWidth under guarded, fully unrolled
// loops.  The last hidden layer is not stored: each of its units is added into the K outputs as soon as it is computed, in
// ascending order, which is the same sum as adding them afterwards.  vec: every row of the second layer's weight starts
// 16 bytes aligned and h1 % 4 == 0, so those rows (the bulk of the parameters) are read 16 bytes at a time
template <int K, int D, bool GLOBAL, int ACT>
__device__ __forceinline__ void mlp_outputs(const float *w, int h1, int h2, bool vec, const float (&o)[D],
                                            float (&z)[K]) {
    const float *b1 = w + h1 * D, *w2 = b1 + h1;
    if (h2 == 0) {
        const float *b2 = w2 + K * h1;
#pragma unroll
        for (int k = 0; k < K; k++) z[k] = mlp_ld<GLOBAL>(b2 + k);
        for (int j = 0; j < h1; j++) {
            float u = mlp_ld<GLOBAL>(b1 + j);
#pragma unroll
            for (int k = 0; k < D; k++) u = u + mlp_ld<GLOBAL>(w + j * D + k) * o[k];
            u = mlp_act<ACT>(u);
#pragma unroll
            for (int k = 0; k < K; k++) z[k] = z[k] + mlp_ld<GLOBAL>(w2 + k * h1 + j) * u;
        }
        return;
    }
    float x[kMlpMaxWidth];
#pragma unroll
    for (int j = 0; j < kMlpMaxWidth; j++) {
        x[j] = 0.0f;
        if (j < h1) {
            float u = mlp_ld<GLOBAL>(b1 + j);
#pragma unroll
            for (int k = 0; k < D; k++) u = u + mlp_ld<GLOBAL>(w + j * D + k) * o[k];
            x[j] = mlp_act<ACT>(u);
        }
    }
    const float *b2 = w2 + h2 * h1, *w3 = b2 + h2, *b3 = w3 + K * h2;
#pragma unroll
    for (int k = 0; k < K; k++) z[k] = mlp_ld<GLOBAL>(b3 + k);
    for (int j = 0; j < h2; j++) {
        const float *row = w2 + j * h1;
        float u = mlp_ld<GLOBAL>(b2 + j);
        if (vec) {
#pragma unroll
            for (int m = 0; m < kMlpMaxWidth; m += 4) {
                if (m < h1) {
                    const float4 q = mlp_ld4<GLOBAL>(row + m);
                    u = u + q.x * x[m];
                    u = u + q.y * x[m + 1];
                    u = u + q.z * x[m + 2];
                    u = u + q.w * x[m + 3];
                }
            }
        } else {
#pragma unroll
            for (int m = 0; m < kMlpMaxWidth; m++)
                if (m < h1) u = u + mlp_ld<GLOBAL>(row + m) * x[m];
        }
        u = mlp_act<ACT>(u);
#pragma unroll
        for (int k = 0; k < K; k++) z[k] = z[k] + mlp_ld<GLOBAL>(w3 + k * h2 + j) * u;
    }
}

// P, the number of floats of one MLP policy D -> h1 (-> h2) -> K: the sum over layers of out * in + out
template <int K, int D>
__host__ __device__ __forceinline__ int64_t mlp_param_count(int64_t h1, int64_t h2) {
    return h2 == 0 ? h1 * D + h1 + K * h1 + K : h1 * D + h1 + h2 * h1 + h2 + K * h2 + K;
}

// The parameters and summary outputs of a b200gym_rollout_mlp launch.  Env i's policy is the P floats at
// params + i * stride; stride 0: one policy shared by every env, which each CTA first copies to shared memory
struct MlpPolicyArgs {
    const float *params;
    int64_t stride;
    int32_t h1, h2;     // hidden widths, h2 = 0 for one hidden layer
    int32_t vec;        // as mlp_outputs
    double *returns;    // [n], SUMMARY only
    int32_t *lengths;
    uint8_t *ended;
};

// MlpActions: LinearActions with the MLP's outputs in place of the logits.  w: the env's parameters, in device memory
// (GLOBAL) or the CTA's shared copy; ACT: the hidden layers' activation (mlp_act)
template <int KIND, bool SUMMARY, bool GLOBAL, int ACT>
struct MlpActions {
    static constexpr int K = linear_logit_count<KIND>(), D = bgym::Env<KIND>::D;
    const float *w;
    int h1, h2;
    bool vec;
    const float (&o)[D];
    template <typename ActT>
    __device__ __forceinline__ ActT action(const ActT *row, int64_t i) const {
        float z[K];
        mlp_outputs<K, D, GLOBAL, ACT>(w, h1, h2, vec, o, z);
        ActT v;
        if constexpr (bgym::Env<KIND>::A == 0) v = (ActT)argmax_first<K>(z);
        else v = z[0];
        if constexpr (!SUMMARY) store_once(const_cast<ActT *>(row) + i, v);
        return v;
    }
};

// T steps of env i under its MLP policy at w (rollout_mlp_kernel): rollout_linear_env's loop, written out again so
// that no pre-existing kernel changes, with MlpActions in place of LinearActions.  The parameters are read at every
// step, from w: a per-env row in device memory (GLOBAL), too large for registers, or the CTA's shared copy.  ACT as
// MlpActions, ReLU when not given
template <int KIND, bool SUMMARY, bool GLOBAL, int ACT = B200GYM_MLP_RELU>
__device__ __forceinline__ void rollout_mlp_env(const StepArgs &a, int64_t i, int32_t T, float *last_obs,
                                                const float *w, const MlpPolicyArgs &p) {
    using E = bgym::Env<KIND>;
    using ActT = typename std::conditional<E::A == 0, long long, float>::type;
    const int64_t n = a.n;
    double s[E::S];
#pragma unroll
    for (int k = 0; k < E::S; k++) s[k] = a.state[k * n + i];
    int32_t elapsed = a.elapsed[i];
    float o[E::D];
    E::observe(s, o);
    const MlpActions<KIND, SUMMARY, GLOBAL, ACT> src{w, p.h1, p.h2, p.vec != 0, o};
    double ret = 0.0;
    int32_t len = 0;
    bool ended = false;
    LinearSink<KIND, SUMMARY> sink{{s, elapsed, a.obs, a.reward, a.terminated, a.truncated, a.final_obs, nullptr},
                                   o, ret, len, ended};
    const ActT *act = reinterpret_cast<const ActT *>(a.actions);
    for (int32_t t = 0; t < T; t++) {
        if (t == T - 1) sink.last = last_obs;
        long long action_int = 0;
        float a0 = 0.0f;
        decode_action<KIND>(src.action(act, i), action_int, a0);
        if (advance_env<KIND>(a, sink, i, s, elapsed, action_int, a0)) reset_env<KIND>(a, sink, i);
        act += n;
        sink.next(n);
    }
#pragma unroll
    for (int k = 0; k < E::S; k++) a.state[k * n + i] = s[k];
    a.elapsed[i] = elapsed;
    if constexpr (SUMMARY) {
        p.returns[i] = ret;
        p.lengths[i] = len;
        p.ended[i] = ended ? 1 : 0;
    }
}

// ---- stochastic rollouts of an MLP policy (b200gym_rollout_mlp_noisy) ---------------------------------------------

// A load of an input the rollout reads once and never again: evict-first on the device, where T steps of noise are far
// larger than L2; a plain load in the host build
template <typename T>
__device__ __forceinline__ T load_once(const T *p) {
#ifdef __CUDA_ARCH__
    return __ldcs(p);
#else
    return *p;
#endif
}

// The arguments of a b200gym_rollout_mlp_noisy launch: the policy (mlp; no summary, so its returns, lengths and ended
// are null) and slice 0 of the [T][n][K] noise it reads and of the [T][n][K] outputs it writes
struct MlpNoisyArgs {
    MlpPolicyArgs mlp;
    const float *noise;
    float *outputs;
};

// y = z + noise[k] for the K outputs z of an MLP, one rounded float32 add each (IEEE: a NaN or infinite term follows
// the sum), with z stored to out[0 .. K-1].  `noise` and `out` point at env i's row
template <int K>
__device__ __forceinline__ void noisy_outputs(const float (&z)[K], const float *noise, float *out, float (&y)[K]) {
    float e[K];
#pragma unroll
    for (int k = 0; k < K; k++) e[k] = load_once(noise + k);
#pragma unroll
    for (int k = 0; k < K; k++) {
        store_once(out + k, z[k]);
        y[k] = z[k] + e[k];
    }
}

// MlpNoisyActions: MlpActions with the caller's noise added to the outputs before the action is taken from them.  The
// outputs z go to `outputs` and the action to the row of actions, both written once; noise and outputs point at row
// t of their [T][n][K] arrays and move on by one row per step (next)
template <int KIND, bool GLOBAL, int ACT>
struct MlpNoisyActions {
    static constexpr int K = linear_logit_count<KIND>(), D = bgym::Env<KIND>::D;
    const float *w;
    int h1, h2;
    bool vec;
    const float (&o)[D];
    const float *noise;
    float *outputs;
    template <typename ActT>
    __device__ __forceinline__ ActT action(const ActT *row, int64_t i) const {
        float z[K], y[K];
        mlp_outputs<K, D, GLOBAL, ACT>(w, h1, h2, vec, o, z);
        noisy_outputs<K>(z, noise + i * K, outputs + i * K, y);
        ActT v;
        if constexpr (bgym::Env<KIND>::A == 0) v = (ActT)argmax_first<K>(y);
        else v = y[0];
        store_once(const_cast<ActT *>(row) + i, v);
        return v;
    }
    __device__ __forceinline__ void next(int64_t n) {
        noise += n * K;
        outputs += n * K;
    }
};

// T steps of env i under its MLP policy at w with the caller's noise (rollout_mlp_noisy_kernel): rollout_mlp_env's
// loop without the summary mode, written out again so that no pre-existing kernel changes, with MlpNoisyActions in
// place of MlpActions; ACT as rollout_mlp_env
template <int KIND, bool GLOBAL, int ACT = B200GYM_MLP_RELU>
__device__ __forceinline__ void rollout_mlp_noisy_env(const StepArgs &a, int64_t i, int32_t T, float *last_obs,
                                                      const float *w, const MlpNoisyArgs &p) {
    using E = bgym::Env<KIND>;
    using ActT = typename std::conditional<E::A == 0, long long, float>::type;
    const int64_t n = a.n;
    double s[E::S];
#pragma unroll
    for (int k = 0; k < E::S; k++) s[k] = a.state[k * n + i];
    int32_t elapsed = a.elapsed[i];
    float o[E::D];
    E::observe(s, o);
    MlpNoisyActions<KIND, GLOBAL, ACT> src{w, p.mlp.h1, p.mlp.h2, p.mlp.vec != 0, o, p.noise, p.outputs};
    double ret = 0.0;
    int32_t len = 0;
    bool ended = false;
    LinearSink<KIND, false> sink{{s, elapsed, a.obs, a.reward, a.terminated, a.truncated, a.final_obs, nullptr},
                                 o, ret, len, ended};
    const ActT *act = reinterpret_cast<const ActT *>(a.actions);
    for (int32_t t = 0; t < T; t++) {
        if (t == T - 1) sink.last = last_obs;
        long long action_int = 0;
        float a0 = 0.0f;
        decode_action<KIND>(src.action(act, i), action_int, a0);
        if (advance_env<KIND>(a, sink, i, s, elapsed, action_int, a0)) reset_env<KIND>(a, sink, i);
        act += n;
        src.next(n);
        sink.next(n);
    }
#pragma unroll
    for (int k = 0; k < E::S; k++) a.state[k * n + i] = s[k];
    a.elapsed[i] = elapsed;
}

// ---- squashed-head MLP rollouts (b200gym_rollout_mlp_head, b200gym_rollout_mlp_noisy_head) -------------------------

// The exp of the SAC head's standard deviation: CUDA's expf on the device, which compiles to the same instructions with
// and without -fmad (DESIGN.md §4.21), and the C library's expf in the host build.  b200gym_selftest_exp evaluates it
__host__ __device__ __forceinline__ float head_exp(float x) { return expf(x); }

// The number of network outputs of head HEAD (b200gym_mlp_head) for a Box action of A dimensions
template <int HEAD>
__host__ __device__ constexpr int head_outputs(int A) {
    static_assert(HEAD == B200GYM_HEAD_TANH || HEAD == B200GYM_HEAD_TANH_NORMAL, "unknown MLP head");
    return HEAD == B200GYM_HEAD_TANH_NORMAL ? 2 * A : A;
}

// The kind's action bounds and CleanRL's action_scale and action_bias from them (b200gym_mlp_head), the same for every
// action dimension of the kinds a head runs on
struct HeadBounds {
    float low, high, scale, bias;
};

// v clamped to [lo, hi] with a NaN staying NaN, as torch.clamp and np.clip do (fminf / fmaxf would drop it)
__host__ __device__ __forceinline__ float head_clamp(float v, float lo, float hi) {
    return v < lo ? lo : (v > hi ? hi : v);
}

// The A actions of head HEAD from the K network outputs z: deterministic (NOISY false; e is not read), or with the
// step's noise e.  Every product and sum is one rounded float32 operation, in the order b200gym_mlp_head gives
template <int HEAD, bool NOISY, int K, int A>
__host__ __device__ __forceinline__ void head_action(const float (&z)[K], const float (&e)[A], const HeadBounds &b,
                                                     float (&act)[A]) {
    static_assert(K == head_outputs<HEAD>(A), "K must be the head's output count");
#pragma unroll
    for (int k = 0; k < A; k++) {
        if constexpr (HEAD == B200GYM_HEAD_TANH_NORMAL && NOISY) {
            const float ls = -5.0f + 3.5f * (mlp_tanh(z[A + k]) + 1.0f);
            const float x = z[k] + e[k] * head_exp(ls);
            act[k] = mlp_tanh(x) * b.scale + b.bias;
        } else {
            const float v = mlp_tanh(z[k]) * b.scale + b.bias;
            if constexpr (NOISY) act[k] = head_clamp(v + e[k], b.low, b.high);
            else act[k] = v;
        }
    }
}

// The arguments of a b200gym_rollout_mlp_head / b200gym_rollout_mlp_noisy_head launch: the policy (mlp), for the noisy
// one slice 0 of the [T][n][A] noise it reads and of the [T][n][K] outputs it writes (null otherwise), and the bounds
struct MlpHeadArgs {
    MlpPolicyArgs mlp;
    const float *noise;
    float *outputs;
    HeadBounds bounds;
};

// MlpHeadActions: MlpActions for a Box kind, with the action taken from the K = head_outputs<HEAD>(A) outputs through
// the deterministic head
template <int KIND, bool SUMMARY, bool GLOBAL, int ACT, int HEAD>
struct MlpHeadActions {
    static constexpr int A = bgym::Env<KIND>::A, K = head_outputs<HEAD>(A), D = bgym::Env<KIND>::D;
    static_assert(A == 1, "the classic Box kinds take one action");
    const float *w;
    int h1, h2;
    bool vec;
    HeadBounds b;
    const float (&o)[D];
    template <typename ActT>
    __device__ __forceinline__ ActT action(const ActT *row, int64_t i) const {
        float z[K], e[A] = {}, y[A];
        mlp_outputs<K, D, GLOBAL, ACT>(w, h1, h2, vec, o, z);
        head_action<HEAD, false>(z, e, b, y);
        const ActT v = y[0];
        if constexpr (!SUMMARY) store_once(const_cast<ActT *>(row) + i, v);
        return v;
    }
};

// MlpNoisyHeadActions: MlpHeadActions with the step's noise (A per env) going into the head.  The outputs z go to
// `outputs` and the action to the row of actions, both written once; noise and outputs point at row t of their
// [T][n][A] and [T][n][K] arrays and move on by one row per step (next)
template <int KIND, bool GLOBAL, int ACT, int HEAD>
struct MlpNoisyHeadActions {
    static constexpr int A = bgym::Env<KIND>::A, K = head_outputs<HEAD>(A), D = bgym::Env<KIND>::D;
    static_assert(A == 1, "the classic Box kinds take one action");
    const float *w;
    int h1, h2;
    bool vec;
    HeadBounds b;
    const float (&o)[D];
    const float *noise;
    float *outputs;
    template <typename ActT>
    __device__ __forceinline__ ActT action(const ActT *row, int64_t i) const {
        float z[K], e[A], y[A];
        mlp_outputs<K, D, GLOBAL, ACT>(w, h1, h2, vec, o, z);
#pragma unroll
        for (int k = 0; k < A; k++) e[k] = load_once(noise + i * A + k);
#pragma unroll
        for (int k = 0; k < K; k++) store_once(outputs + i * K + k, z[k]);
        head_action<HEAD, true>(z, e, b, y);
        const ActT v = y[0];
        store_once(const_cast<ActT *>(row) + i, v);
        return v;
    }
    __device__ __forceinline__ void next(int64_t n) {
        noise += n * A;
        outputs += n * K;
    }
};

// T steps of env i under its MLP policy at w through head HEAD (rollout_mlp_head_kernel): rollout_mlp_env's loop,
// written out again so that no pre-existing kernel changes, with MlpHeadActions in place of MlpActions; SUMMARY,
// GLOBAL and ACT as rollout_mlp_env
template <int KIND, bool SUMMARY, bool GLOBAL, int ACT, int HEAD>
__device__ __forceinline__ void rollout_mlp_head_env(const StepArgs &a, int64_t i, int32_t T, float *last_obs,
                                                     const float *w, const MlpHeadArgs &p) {
    using E = bgym::Env<KIND>;
    const int64_t n = a.n;
    double s[E::S];
#pragma unroll
    for (int k = 0; k < E::S; k++) s[k] = a.state[k * n + i];
    int32_t elapsed = a.elapsed[i];
    float o[E::D];
    E::observe(s, o);
    const MlpHeadActions<KIND, SUMMARY, GLOBAL, ACT, HEAD> src{w, p.mlp.h1, p.mlp.h2, p.mlp.vec != 0, p.bounds, o};
    double ret = 0.0;
    int32_t len = 0;
    bool ended = false;
    LinearSink<KIND, SUMMARY> sink{{s, elapsed, a.obs, a.reward, a.terminated, a.truncated, a.final_obs, nullptr},
                                   o, ret, len, ended};
    const float *act = reinterpret_cast<const float *>(a.actions);
    for (int32_t t = 0; t < T; t++) {
        if (t == T - 1) sink.last = last_obs;
        long long action_int = 0;
        float a0 = 0.0f;
        decode_action<KIND>(src.action(act, i), action_int, a0);
        if (advance_env<KIND>(a, sink, i, s, elapsed, action_int, a0)) reset_env<KIND>(a, sink, i);
        act += n;
        sink.next(n);
    }
#pragma unroll
    for (int k = 0; k < E::S; k++) a.state[k * n + i] = s[k];
    a.elapsed[i] = elapsed;
    if constexpr (SUMMARY) {
        p.mlp.returns[i] = ret;
        p.mlp.lengths[i] = len;
        p.mlp.ended[i] = ended ? 1 : 0;
    }
}

// T steps of env i under its MLP policy at w with the caller's noise through head HEAD
// (rollout_mlp_noisy_head_kernel): rollout_mlp_noisy_env's loop, written out again so that no pre-existing kernel
// changes, with MlpNoisyHeadActions in place of MlpNoisyActions; GLOBAL and ACT as rollout_mlp_env
template <int KIND, bool GLOBAL, int ACT, int HEAD>
__device__ __forceinline__ void rollout_mlp_noisy_head_env(const StepArgs &a, int64_t i, int32_t T, float *last_obs,
                                                           const float *w, const MlpHeadArgs &p) {
    using E = bgym::Env<KIND>;
    const int64_t n = a.n;
    double s[E::S];
#pragma unroll
    for (int k = 0; k < E::S; k++) s[k] = a.state[k * n + i];
    int32_t elapsed = a.elapsed[i];
    float o[E::D];
    E::observe(s, o);
    MlpNoisyHeadActions<KIND, GLOBAL, ACT, HEAD> src{w, p.mlp.h1, p.mlp.h2, p.mlp.vec != 0, p.bounds, o, p.noise,
                                                     p.outputs};
    double ret = 0.0;
    int32_t len = 0;
    bool ended = false;
    LinearSink<KIND, false> sink{{s, elapsed, a.obs, a.reward, a.terminated, a.truncated, a.final_obs, nullptr},
                                 o, ret, len, ended};
    const float *act = reinterpret_cast<const float *>(a.actions);
    for (int32_t t = 0; t < T; t++) {
        if (t == T - 1) sink.last = last_obs;
        long long action_int = 0;
        float a0 = 0.0f;
        decode_action<KIND>(src.action(act, i), action_int, a0);
        if (advance_env<KIND>(a, sink, i, s, elapsed, action_int, a0)) reset_env<KIND>(a, sink, i);
        act += n;
        src.next(n);
        sink.next(n);
    }
#pragma unroll
    for (int k = 0; k < E::S; k++) a.state[k * n + i] = s[k];
    a.elapsed[i] = elapsed;
}

// ---- on-policy collection with a critic (b200gym_rollout_actor_critic) --------------------------------------------

// The arguments of a b200gym_rollout_actor_critic launch: the actor and its noise and outputs (one actor shared by every
// env, so actor.mlp.stride is 0), the critic (the actor's widths, one output), and slice 0 of the [T + 1][n] values and
// of the [T][n] advantages.  Until gae_kernel runs, advantages[t][i] holds V(final observation) where step t of env i
// truncated without terminating, and nothing anywhere else
struct ActorCriticArgs {
    MlpNoisyArgs actor;
    const float *critic;
    float *values;
    float *advantages;
};

// The sink of an actor-critic rollout: LinearSink's, plus a register copy of the step's flags and of its final
// observation, from which the driver evaluates the critic where the step truncated without terminating
template <int KIND>
struct CriticSink : LinearSink<KIND, false> {
    using Base = LinearSink<KIND, false>;
    float (&fin)[bgym::Env<KIND>::D];
    uint8_t &te, &tr;
    template <typename I>
    __device__ __forceinline__ void scalars(I i, double reward, uint8_t term, uint8_t trunc) const {
        Base::scalars(i, reward, term, trunc);
        te = term;
        tr = trunc;
    }
    template <int D, typename I>
    __device__ __forceinline__ void final_obs(I i, const float (&v)[D]) const {
        Base::template final_obs<D>(i, v);
#pragma unroll
        for (int k = 0; k < D; k++) fin[k] = v[k];
    }
};

// T steps of env i under the noisy actor at wa with the critic at wc (rollout_actor_critic_kernel): rollout_mlp_noisy_env's
// loop, written out again so that no pre-existing kernel changes, with the critic evaluated at every step on the
// observation the actor reads, V(o) stored to values[t], and on the final observation of a step that truncated without
// terminating, V stored to the holding slot advantages[t][i].  After the loop, values[T] = V(the observation the call
// leaves the env at).  The caller's autoreset must be on: the bootstrap reads the final observations.  wa and wc are
// the CTA's shared copies (mlp_stage_pair), so both nets read the same widths and the same vec
template <int KIND, int ACT = B200GYM_MLP_RELU>
__device__ __forceinline__ void rollout_actor_critic_env(const StepArgs &a, int64_t i, int32_t T, float *last_obs,
                                                         const float *wa, const float *wc, const ActorCriticArgs &p) {
    using E = bgym::Env<KIND>;
    using ActT = typename std::conditional<E::A == 0, long long, float>::type;
    const int64_t n = a.n;
    const int h1 = p.actor.mlp.h1, h2 = p.actor.mlp.h2;
    const bool vec = p.actor.mlp.vec != 0;
    double s[E::S];
#pragma unroll
    for (int k = 0; k < E::S; k++) s[k] = a.state[k * n + i];
    int32_t elapsed = a.elapsed[i];
    float o[E::D], fin[E::D];
    E::observe(s, o);
    MlpNoisyActions<KIND, false, ACT> src{wa, h1, h2, vec, o, p.actor.noise, p.actor.outputs};
    double ret = 0.0;
    int32_t len = 0;
    bool ended = false;
    uint8_t te = 0, tr = 0;
    CriticSink<KIND> sink{{{s, elapsed, a.obs, a.reward, a.terminated, a.truncated, a.final_obs, nullptr},
                           o, ret, len, ended},
                          fin, te, tr};
    const ActT *act = reinterpret_cast<const ActT *>(a.actions);
    float *values = p.values, *held = p.advantages;
    for (int32_t t = 0; t < T; t++) {
        if (t == T - 1) sink.last = last_obs;
        float v[1];
        mlp_outputs<1, E::D, false, ACT>(wc, h1, h2, vec, o, v);
        store_once(values + i, v[0]);
        long long action_int = 0;
        float a0 = 0.0f;
        decode_action<KIND>(src.action(act, i), action_int, a0);
        if (advance_env<KIND>(a, sink, i, s, elapsed, action_int, a0)) reset_env<KIND>(a, sink, i);
        if (tr && !te) {
            mlp_outputs<1, E::D, false, ACT>(wc, h1, h2, vec, fin, v);
            store_once(held + i, v[0]);
        }
        act += n;
        values += n;
        held += n;
        src.next(n);
        sink.next(n);
    }
    float v[1];
    mlp_outputs<1, E::D, false, ACT>(wc, h1, h2, vec, o, v);
    store_once(values + i, v[0]);
#pragma unroll
    for (int k = 0; k < E::S; k++) a.state[k * n + i] = s[k];
    a.elapsed[i] = elapsed;
}

// The GAE recursion of env i over the T steps of a b200gym_rollout_actor_critic call (gae_kernel), in float32, every
// operation rounded, no fused multiply-add (the library is built with -fmad=false, the host build with
// -ffp-contract=off), with g = gamma and gl = gamma * gae_lambda already rounded to float32:
//   r = (float)reward[t]; adv[T] = +0.0; for t = T-1 .. 0:
//   terminated: delta = r - V[t]; else truncated: delta = (r + g * Vf[t]) - V[t]; else delta = (r + g * V[t+1]) - V[t]
//   adv[t] = delta if terminated or truncated, else delta + gl * adv[t+1]
// Vf[t] is read from adv's own slot t (rollout_actor_critic_env leaves it there), which the step then overwrites.  All
// arrays are [T][n] but values, [T + 1][n]
__host__ __device__ __forceinline__ void gae_env(int64_t i, int64_t n, int32_t T, float g, float gl,
                                                 const double *reward, const uint8_t *term, const uint8_t *trunc,
                                                 const float *values, float *adv) {
    float next = 0.0f;
    for (int32_t t = T - 1; t >= 0; t--) {
        const int64_t k = (int64_t)t * n + i;
        const float r = (float)reward[k], v = values[k];
        const bool te = term[k] != 0, tr = trunc[k] != 0;
        float delta;
        if (te) delta = r - v;
        else if (tr) delta = (r + g * adv[k]) - v;
        else delta = (r + g * values[k + n]) - v;
        next = (te || tr) ? delta : delta + gl * next;
        adv[k] = next;
    }
}

// ---- normalised observations and rewards (b200gym_rollout_mlp_noisy_norm, b200gym_rollout_actor_critic_norm) ------

// The standard deviation of one column of a running variance, sqrt(var + eps) in float64 (normalize.py:94)
__host__ __device__ __forceinline__ double norm_sd(double var, double eps) { return sqrt(var + eps); }

// One normalised observation element: float32((float64(o) - mean) / sd), rms_apply_kernel's expression, then clamped to
// [-clip, clip] with torch.clamp's bits: a NaN stays NaN, -0.0 stays -0.0, and clip = +inf clamps nothing
__host__ __device__ __forceinline__ float norm_obs_elem(float o, double mean, double sd, float clip) {
    const float x = (float)(((double)o - mean) / sd);
    return x < -clip ? -clip : (x > clip ? clip : x);
}

// The network input x of observation o: norm_obs_elem per element, with mean[D] and sd[D] the CTA's shared copies
template <int D>
__host__ __device__ __forceinline__ void norm_obs(const float (&o)[D], const double *mean, const double *sd, float clip,
                                                  float (&x)[D]) {
#pragma unroll
    for (int k = 0; k < D; k++) x[k] = norm_obs_elem(o[k], mean[k], sd[k], clip);
}

// The statistics a normalising launch reads, all fixed for the call: the observations' mean[D] and var[D] (float64,
// caller-owned; staged with norm_sd once per CTA), eps, and the clip (+inf: none)
struct ObsNormArgs {
    const double *mean, *var;
    double eps;
    float clip;
};

// T steps of env i under the shared noisy policy at w with normalised inputs (rollout_mlp_noisy_norm_kernel):
// rollout_mlp_noisy_env's loop, written out again so that no pre-existing kernel changes, with the policy reading x,
// norm_obs of the observation o, in place of o.  o stays raw, so the sink stores the raw observations.  mean and sd are
// the CTA's shared copies
template <int KIND, int ACT = B200GYM_MLP_RELU>
__device__ __forceinline__ void rollout_mlp_noisy_norm_env(const StepArgs &a, int64_t i, int32_t T, float *last_obs,
                                                           const float *w, const MlpNoisyArgs &p, const double *mean,
                                                           const double *sd, float clip) {
    using E = bgym::Env<KIND>;
    using ActT = typename std::conditional<E::A == 0, long long, float>::type;
    const int64_t n = a.n;
    double s[E::S];
#pragma unroll
    for (int k = 0; k < E::S; k++) s[k] = a.state[k * n + i];
    int32_t elapsed = a.elapsed[i];
    float o[E::D], x[E::D];
    E::observe(s, o);
    norm_obs<E::D>(o, mean, sd, clip, x);
    MlpNoisyActions<KIND, false, ACT> src{w, p.mlp.h1, p.mlp.h2, p.mlp.vec != 0, x, p.noise, p.outputs};
    double ret = 0.0;
    int32_t len = 0;
    bool ended = false;
    LinearSink<KIND, false> sink{{s, elapsed, a.obs, a.reward, a.terminated, a.truncated, a.final_obs, nullptr},
                                 o, ret, len, ended};
    const ActT *act = reinterpret_cast<const ActT *>(a.actions);
    for (int32_t t = 0; t < T; t++) {
        if (t == T - 1) sink.last = last_obs;
        long long action_int = 0;
        float a0 = 0.0f;
        decode_action<KIND>(src.action(act, i), action_int, a0);
        if (advance_env<KIND>(a, sink, i, s, elapsed, action_int, a0)) reset_env<KIND>(a, sink, i);
        norm_obs<E::D>(o, mean, sd, clip, x);
        act += n;
        src.next(n);
        sink.next(n);
    }
#pragma unroll
    for (int k = 0; k < E::S; k++) a.state[k * n + i] = s[k];
    a.elapsed[i] = elapsed;
}

// T steps of env i under the noisy actor at wa with the critic at wc, both reading normalised inputs
// (rollout_actor_critic_norm_kernel): rollout_actor_critic_env's loop, written out again so that no pre-existing kernel
// changes, with the actor and the critic reading x = norm_obs(o) in place of o, and the truncation bootstrap reading
// norm_obs of the final observation.  o and the final observation stay raw for the sink
template <int KIND, int ACT = B200GYM_MLP_RELU>
__device__ __forceinline__ void rollout_actor_critic_norm_env(const StepArgs &a, int64_t i, int32_t T, float *last_obs,
                                                              const float *wa, const float *wc,
                                                              const ActorCriticArgs &p, const double *mean,
                                                              const double *sd, float clip) {
    using E = bgym::Env<KIND>;
    using ActT = typename std::conditional<E::A == 0, long long, float>::type;
    const int64_t n = a.n;
    const int h1 = p.actor.mlp.h1, h2 = p.actor.mlp.h2;
    const bool vec = p.actor.mlp.vec != 0;
    double s[E::S];
#pragma unroll
    for (int k = 0; k < E::S; k++) s[k] = a.state[k * n + i];
    int32_t elapsed = a.elapsed[i];
    float o[E::D], x[E::D], fin[E::D];
    E::observe(s, o);
    norm_obs<E::D>(o, mean, sd, clip, x);
    MlpNoisyActions<KIND, false, ACT> src{wa, h1, h2, vec, x, p.actor.noise, p.actor.outputs};
    double ret = 0.0;
    int32_t len = 0;
    bool ended = false;
    uint8_t te = 0, tr = 0;
    CriticSink<KIND> sink{{{s, elapsed, a.obs, a.reward, a.terminated, a.truncated, a.final_obs, nullptr},
                           o, ret, len, ended},
                          fin, te, tr};
    const ActT *act = reinterpret_cast<const ActT *>(a.actions);
    float *values = p.values, *held = p.advantages;
    for (int32_t t = 0; t < T; t++) {
        if (t == T - 1) sink.last = last_obs;
        float v[1];
        mlp_outputs<1, E::D, false, ACT>(wc, h1, h2, vec, x, v);
        store_once(values + i, v[0]);
        long long action_int = 0;
        float a0 = 0.0f;
        decode_action<KIND>(src.action(act, i), action_int, a0);
        if (advance_env<KIND>(a, sink, i, s, elapsed, action_int, a0)) reset_env<KIND>(a, sink, i);
        if (tr && !te) {
            norm_obs<E::D>(fin, mean, sd, clip, fin);
            mlp_outputs<1, E::D, false, ACT>(wc, h1, h2, vec, fin, v);
            store_once(held + i, v[0]);
        }
        norm_obs<E::D>(o, mean, sd, clip, x);
        act += n;
        values += n;
        held += n;
        src.next(n);
        sink.next(n);
    }
    float v[1];
    mlp_outputs<1, E::D, false, ACT>(wc, h1, h2, vec, x, v);
    store_once(values + i, v[0]);
#pragma unroll
    for (int k = 0; k < E::S; k++) a.state[k * n + i] = s[k];
    a.elapsed[i] = elapsed;
}

// gae_env with scaled rewards (gae_scaled_kernel): r = float32(reward[t] / sd), then clamped to [-clip, clip] as
// norm_obs_elem clamps (clip = +inf: none), in place of r = (float)reward[t]; sd = norm_sd of the return variance.
// Written out again so that gae_env and gae_kernel keep their code
__host__ __device__ __forceinline__ void gae_scaled_env(int64_t i, int64_t n, int32_t T, float g, float gl, double sd,
                                                        float clip, const double *reward, const uint8_t *term,
                                                        const uint8_t *trunc, const float *values, float *adv) {
    float next = 0.0f;
    for (int32_t t = T - 1; t >= 0; t--) {
        const int64_t k = (int64_t)t * n + i;
        const float q = (float)(reward[k] / sd), v = values[k];
        const float r = q < -clip ? -clip : (q > clip ? clip : q);
        const bool te = term[k] != 0, tr = trunc[k] != 0;
        float delta;
        if (te) delta = r - v;
        else if (tr) delta = (r + g * adv[k]) - v;
        else delta = (r + g * values[k + n]) - v;
        next = (te || tr) ? delta : delta + gl * next;
        adv[k] = next;
    }
}

// ---- normalised inputs and observation moments in the closed-loop rollouts (b200gym_rollout_linear_norm,
// b200gym_rollout_mlp_norm) ----------------------------------------------------------------------------------------

// The observation moments of a summary-mode rollout: env i's rows sum[i][D] and sumsq[i][D], float64; both null: none
struct ObsMomentArgs {
    double *sum, *sumsq;
};

// The policy's input x of observation o: norm_obs with the CTA's shared statistics, or o itself where the rollout is
// not normalised (mean null, the same for every thread of the launch)
template <int D>
__host__ __device__ __forceinline__ void norm_obs_or_raw(const float (&o)[D], const double *mean, const double *sd,
                                                         float clip, float (&x)[D]) {
    if (mean) {
        norm_obs<D>(o, mean, sd, clip, x);
    } else {
#pragma unroll
        for (int k = 0; k < D; k++) x[k] = o[k];
    }
}

// One step of the observation moments: s[k] = s[k] + float64(o[k]) and q[k] = q[k] + float64(o[k]) * float64(o[k]),
// every operation rounded (no fused multiply-add: -fmad=false on the device, -ffp-contract=off in the host build)
template <int D>
__host__ __device__ __forceinline__ void moments_fold(const float (&o)[D], double (&s)[D], double (&q)[D]) {
#pragma unroll
    for (int k = 0; k < D; k++) {
        const double v = (double)o[k];
        s[k] = s[k] + v;
        q[k] = q[k] + v * v;
    }
}

// T steps of env i under its linear policy with normalised inputs (rollout_linear_norm_kernel): rollout_linear_env's
// loop, written out again so that no pre-existing kernel changes, with the policy reading x = norm_obs_or_raw(o) in
// place of o, computed at the top of each step so that only o is live across the step.  o stays raw, so the sink
// stores the raw observations.  SUMMARY with m.sum not null: the moments of the raw inputs of steps 0 .. len - 1 (the
// first episode's), folded in step order from +0.0 before each step's action while the episode has not ended, then
// stored to env i's rows
template <int KIND, bool SUMMARY>
__device__ __forceinline__ void rollout_linear_norm_env(const StepArgs &a, int64_t i, int32_t T, float *last_obs,
                                                        const LinearPolicyArgs &p, const double *mean, const double *sd,
                                                        float clip, const ObsMomentArgs &m) {
    using E = bgym::Env<KIND>;
    using ActT = typename std::conditional<E::A == 0, long long, float>::type;
    using Src = LinearActions<KIND, SUMMARY>;
    const int64_t n = a.n;
    double s[E::S];
#pragma unroll
    for (int k = 0; k < E::S; k++) s[k] = a.state[k * n + i];
    int32_t elapsed = a.elapsed[i];
    float o[E::D], x[E::D];
    E::observe(s, o);
    Src src{{}, {}, x};
    const float *w = p.weight + i * p.w_stride, *b = p.bias + i * p.b_stride;
#pragma unroll
    for (int k = 0; k < Src::K * E::D; k++) src.w[k] = __ldg(w + k);
#pragma unroll
    for (int j = 0; j < Src::K; j++) src.b[j] = __ldg(b + j);
    double ret = 0.0;
    int32_t len = 0;
    bool ended = false;
    const bool moments = SUMMARY && m.sum != nullptr;
    double ms[E::D], mq[E::D];
#pragma unroll
    for (int k = 0; k < E::D; k++) ms[k] = mq[k] = 0.0;
    LinearSink<KIND, SUMMARY> sink{{s, elapsed, a.obs, a.reward, a.terminated, a.truncated, a.final_obs, nullptr},
                                   o, ret, len, ended};
    const ActT *act = reinterpret_cast<const ActT *>(a.actions);
    for (int32_t t = 0; t < T; t++) {
        if (t == T - 1) sink.last = last_obs;
        if (moments && !ended) moments_fold<E::D>(o, ms, mq);
        norm_obs_or_raw<E::D>(o, mean, sd, clip, x);
        long long action_int = 0;
        float a0 = 0.0f;
        decode_action<KIND>(src.action(act, i), action_int, a0);
        if (advance_env<KIND>(a, sink, i, s, elapsed, action_int, a0)) reset_env<KIND>(a, sink, i);
        act += n;
        sink.next(n);
    }
#pragma unroll
    for (int k = 0; k < E::S; k++) a.state[k * n + i] = s[k];
    a.elapsed[i] = elapsed;
    if constexpr (SUMMARY) {
        p.returns[i] = ret;
        p.lengths[i] = len;
        p.ended[i] = ended ? 1 : 0;
        if (moments) {
#pragma unroll
            for (int k = 0; k < E::D; k++) {
                m.sum[i * E::D + k] = ms[k];
                m.sumsq[i * E::D + k] = mq[k];
            }
        }
    }
}

// T steps of env i under its MLP policy at w with normalised inputs (rollout_mlp_norm_kernel): rollout_mlp_env's loop,
// written out again so that no pre-existing kernel changes, with MlpActions reading x = norm_obs_or_raw(o) in place of
// o; the moments as rollout_linear_norm_env's.  GLOBAL and ACT as rollout_mlp_env
template <int KIND, bool SUMMARY, bool GLOBAL, int ACT>
__device__ __forceinline__ void rollout_mlp_norm_env(const StepArgs &a, int64_t i, int32_t T, float *last_obs,
                                                     const float *w, const MlpPolicyArgs &p, const double *mean,
                                                     const double *sd, float clip, const ObsMomentArgs &m) {
    using E = bgym::Env<KIND>;
    using ActT = typename std::conditional<E::A == 0, long long, float>::type;
    const int64_t n = a.n;
    double s[E::S];
#pragma unroll
    for (int k = 0; k < E::S; k++) s[k] = a.state[k * n + i];
    int32_t elapsed = a.elapsed[i];
    float o[E::D], x[E::D];
    E::observe(s, o);
    const MlpActions<KIND, SUMMARY, GLOBAL, ACT> src{w, p.h1, p.h2, p.vec != 0, x};
    double ret = 0.0;
    int32_t len = 0;
    bool ended = false;
    const bool moments = SUMMARY && m.sum != nullptr;
    double ms[E::D], mq[E::D];
#pragma unroll
    for (int k = 0; k < E::D; k++) ms[k] = mq[k] = 0.0;
    LinearSink<KIND, SUMMARY> sink{{s, elapsed, a.obs, a.reward, a.terminated, a.truncated, a.final_obs, nullptr},
                                   o, ret, len, ended};
    const ActT *act = reinterpret_cast<const ActT *>(a.actions);
    for (int32_t t = 0; t < T; t++) {
        if (t == T - 1) sink.last = last_obs;
        if (moments && !ended) moments_fold<E::D>(o, ms, mq);
        norm_obs_or_raw<E::D>(o, mean, sd, clip, x);
        long long action_int = 0;
        float a0 = 0.0f;
        decode_action<KIND>(src.action(act, i), action_int, a0);
        if (advance_env<KIND>(a, sink, i, s, elapsed, action_int, a0)) reset_env<KIND>(a, sink, i);
        act += n;
        sink.next(n);
    }
#pragma unroll
    for (int k = 0; k < E::S; k++) a.state[k * n + i] = s[k];
    a.elapsed[i] = elapsed;
    if constexpr (SUMMARY) {
        p.returns[i] = ret;
        p.lengths[i] = len;
        p.ended[i] = ended ? 1 : 0;
        if (moments) {
#pragma unroll
            for (int k = 0; k < E::D; k++) {
                m.sum[i * E::D + k] = ms[k];
                m.sumsq[i * E::D + k] = mq[k];
            }
        }
    }
}

// ---- rollouts from snapshot rows (b200gym_rollout_from) ------------------------------------------------------------

// The snapshot row of a classic kind (b200gym.cu, snapshot_save_kernel): the PCG64 record {state_hi, state_lo, inc_hi,
// inc_lo} in bytes [0, 32), float64 state[S] from byte 32, then the TimeLimit counter, the flag byte in the low byte of
// the next word, and zeros up to a multiple of 32 bytes
template <int KIND>
__host__ __device__ constexpr int classic_row_bytes() {
    return (32 + 8 * bgym::Env<KIND>::S + 4 + 1 + 31) / 32 * 32;
}

// The arguments of a b200gym_rollout_from launch.  Branch b starts from row row_idx[b] (row_idx null: row b) of the
// n_rows rows at `rows`; a row index out of range skips the branch: zero outputs, and `bad` raised.  end_rows and
// end_obs: null, or [B] rows and observations of the end states (STATES)
struct RolloutFromArgs {
    const unsigned char *rows;
    int64_t n_rows;
    const int64_t *row_idx;
    double *returns;
    int32_t *lengths;
    uint8_t *ended;
    unsigned char *end_rows;
    float *end_obs;
    unsigned long long *bad;   // page-locked, device-mapped word (the handle's snapshot index-error flag)
};

// T steps of branch b (rollout_from_kernel): rollout_env's loop from a snapshot row instead of the handle's arrays,
// written out again so that no pre-existing kernel changes.  The PCG64 stream of the autoresets, the state and the
// TimeLimit counter are loaded from the row once and held in registers (reset_env_from, never reset_env: the handle's
// records are not the branch's).  a.actions is the [T][B] array and a.n = B; a.flags[f] is the branch's own copy of
// the row's flag byte, which advance_env reads and writes for CartPole without autoreset (the kernel gives each thread
// a byte of shared memory; nothing else is indexed by f).  LinearSink<KIND, true> folds the rewards and flags into the
// episode summary and keeps the last observation; nothing is stored per step.  STATES: the end row in the layout of
// classic_row_bytes and the end observation are stored at the end
template <int KIND, typename ActT, bool STATES, typename I>
__device__ __forceinline__ void rollout_from_env(const StepArgs &a, int64_t b, I f, int32_t T,
                                                 const RolloutFromArgs &p) {
    using E = bgym::Env<KIND>;
    constexpr int R = classic_row_bytes<KIND>(), C = R / 16;
    const int64_t row = p.row_idx ? p.row_idx[b] : b;
    if (row < 0 || row >= p.n_rows) {
        *reinterpret_cast<volatile unsigned long long *>(p.bad) = 1ULL;
        p.returns[b] = 0.0;
        p.lengths[b] = 0;
        p.ended[b] = 0;
        if constexpr (STATES) {
            ulonglong2 *out = reinterpret_cast<ulonglong2 *>(p.end_rows + b * R);
#pragma unroll
            for (int c = 0; c < C; c++) out[c] = make_ulonglong2(0ULL, 0ULL);
#pragma unroll
            for (int k = 0; k < E::D; k++) p.end_obs[b * E::D + k] = 0.0f;
        }
        return;
    }
    const ulonglong2 *in = reinterpret_cast<const ulonglong2 *>(p.rows + row * R);
    bgym::Pcg64 g = bgym::pcg64_load(reinterpret_cast<const uint64_t *>(in));
    double s[E::S];
#pragma unroll
    for (int k = 0; k < E::S; k += 2) {
        const ulonglong2 v = __ldg(in + 2 + k / 2);
        s[k] = __longlong_as_double((long long)v.x);
        s[k + 1] = __longlong_as_double((long long)v.y);
    }
    const ulonglong2 tail = __ldg(in + 2 + E::S / 2);   // {elapsed | flags << 32, 0}
    int32_t elapsed = (int32_t)(uint32_t)tail.x;
    a.flags[f] = (uint8_t)(tail.x >> 32);
    float o[E::D] = {};
    double ret = 0.0;
    int32_t len = 0;
    bool ended = false;
    LinearSink<KIND, true> sink{{s, elapsed, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr}, o, ret, len, ended};
    const ActT *act = reinterpret_cast<const ActT *>(a.actions);
    const ReadActions src{};
    for (int32_t t = 0; t < T; t++) {
        long long action_int = 0;
        float a0 = 0.0f;
        decode_action<KIND>(src.action(act, b), action_int, a0);
        if (advance_env<KIND>(a, sink, f, s, elapsed, action_int, a0)) reset_env_from<KIND>(sink, f, g);
        act += a.n;
    }
    p.returns[b] = ret;
    p.lengths[b] = len;
    p.ended[b] = ended ? 1 : 0;
    if constexpr (STATES) {
        static_assert(E::S % 2 == 0 && 2 + E::S / 2 + 1 <= C, "row layout");
        ulonglong2 *out = reinterpret_cast<ulonglong2 *>(p.end_rows + b * R);
        out[0] = make_ulonglong2((unsigned long long)(uint64_t)(g.state >> 64), (unsigned long long)(uint64_t)g.state);
        out[1] = make_ulonglong2((unsigned long long)(uint64_t)(g.inc >> 64), (unsigned long long)(uint64_t)g.inc);
#pragma unroll
        for (int k = 0; k < E::S; k += 2)
            out[2 + k / 2] = make_ulonglong2((unsigned long long)__double_as_longlong(s[k]),
                                             (unsigned long long)__double_as_longlong(s[k + 1]));
        out[2 + E::S / 2] = make_ulonglong2((unsigned long long)(uint32_t)elapsed |
                                                ((unsigned long long)a.flags[f] << 32), 0ULL);
#pragma unroll
        for (int c = 2 + E::S / 2 + 1; c < C; c++) out[c] = make_ulonglong2(0ULL, 0ULL);
        store_row<E::D>(p.end_obs, b, o);
    }
}

// ---- closed-loop MLP-policy rollouts from snapshot rows (b200gym_rollout_from_mlp) ---------------------------------

// The arguments of a b200gym_rollout_from_mlp launch: the rows, outputs and end states as rollout_from's (from), the
// policy (mlp: branch b's parameters are params + b * stride; no summary pointers), the noise (null: none; otherwise
// slice 0 of [T][B][K]) and the action each branch took at step 0, [B] long long (Discrete) or [B][A] float (Box)
struct RolloutFromMlpArgs {
    RolloutFromArgs from;
    MlpPolicyArgs mlp;
    const float *noise;
    void *first_actions;
};

// T steps of branch b under its MLP policy at w (rollout_from_mlp_kernel): rollout_from_env's row load, flag byte and
// end row with rollout_mlp_env's policy step, written out again so that no pre-existing kernel changes.  Step 0's
// input is observe() of the row's state, as rollout_mlp_env's is of the env's.  The policy reads x = norm_obs_or_raw(o)
// (mean null: o itself); with noise, the action is taken from z + noise[t][b] (noisy_outputs' adds, without its
// stores), and without, from z itself, so the deterministic actions are rollout_mlp_env's bits.  Both choices are the
// same for every thread of the launch.  Nothing is stored per step but the action of step 0; a skipped branch gets
// zeros.  GLOBAL and ACT as rollout_mlp_env, STATES as rollout_from_env
template <int KIND, bool STATES, bool GLOBAL, int ACT, typename I>
__device__ __forceinline__ void rollout_from_mlp_env(const StepArgs &a, int64_t b, I f, int32_t T, const float *w,
                                                     const RolloutFromMlpArgs &p, const double *mean, const double *sd,
                                                     float clip) {
    using E = bgym::Env<KIND>;
    using ActT = typename std::conditional<E::A == 0, long long, float>::type;
    constexpr int K = MlpActions<KIND, true, GLOBAL, ACT>::K, R = classic_row_bytes<KIND>(), C = R / 16;
    static_assert(E::A <= 1, "one action element per branch");
    const RolloutFromArgs &q = p.from;
    ActT *first = static_cast<ActT *>(p.first_actions);
    const int64_t row = q.row_idx ? q.row_idx[b] : b;
    if (row < 0 || row >= q.n_rows) {
        *reinterpret_cast<volatile unsigned long long *>(q.bad) = 1ULL;
        q.returns[b] = 0.0;
        q.lengths[b] = 0;
        q.ended[b] = 0;
        first[b] = (ActT)0;
        if constexpr (STATES) {
            ulonglong2 *out = reinterpret_cast<ulonglong2 *>(q.end_rows + b * R);
#pragma unroll
            for (int c = 0; c < C; c++) out[c] = make_ulonglong2(0ULL, 0ULL);
#pragma unroll
            for (int k = 0; k < E::D; k++) q.end_obs[b * E::D + k] = 0.0f;
        }
        return;
    }
    const ulonglong2 *in = reinterpret_cast<const ulonglong2 *>(q.rows + row * R);
    bgym::Pcg64 g = bgym::pcg64_load(reinterpret_cast<const uint64_t *>(in));
    double s[E::S];
#pragma unroll
    for (int k = 0; k < E::S; k += 2) {
        const ulonglong2 v = __ldg(in + 2 + k / 2);
        s[k] = __longlong_as_double((long long)v.x);
        s[k + 1] = __longlong_as_double((long long)v.y);
    }
    const ulonglong2 tail = __ldg(in + 2 + E::S / 2);   // {elapsed | flags << 32, 0}
    int32_t elapsed = (int32_t)(uint32_t)tail.x;
    a.flags[f] = (uint8_t)(tail.x >> 32);
    float o[E::D], x[E::D];
    E::observe(s, o);
    const int h1 = p.mlp.h1, h2 = p.mlp.h2;
    const bool vec = p.mlp.vec != 0;
    const float *noise = p.noise ? p.noise + b * K : nullptr;
    double ret = 0.0;
    int32_t len = 0;
    bool ended = false;
    LinearSink<KIND, true> sink{{s, elapsed, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr}, o, ret, len, ended};
    for (int32_t t = 0; t < T; t++) {
        norm_obs_or_raw<E::D>(o, mean, sd, clip, x);
        float z[K];
        mlp_outputs<K, E::D, GLOBAL, ACT>(w, h1, h2, vec, x, z);
        if (noise) {
            float e[K];
#pragma unroll
            for (int k = 0; k < K; k++) e[k] = load_once(noise + k);
#pragma unroll
            for (int k = 0; k < K; k++) z[k] = z[k] + e[k];
            noise += a.n * K;
        }
        ActT v;
        if constexpr (E::A == 0) v = (ActT)argmax_first<K>(z);
        else v = z[0];
        if (t == 0) first[b] = v;
        long long action_int = 0;
        float a0 = 0.0f;
        decode_action<KIND>(v, action_int, a0);
        if (advance_env<KIND>(a, sink, f, s, elapsed, action_int, a0)) reset_env_from<KIND>(sink, f, g);
    }
    q.returns[b] = ret;
    q.lengths[b] = len;
    q.ended[b] = ended ? 1 : 0;
    if constexpr (STATES) {
        static_assert(E::S % 2 == 0 && 2 + E::S / 2 + 1 <= C, "row layout");
        ulonglong2 *out = reinterpret_cast<ulonglong2 *>(q.end_rows + b * R);
        out[0] = make_ulonglong2((unsigned long long)(uint64_t)(g.state >> 64), (unsigned long long)(uint64_t)g.state);
        out[1] = make_ulonglong2((unsigned long long)(uint64_t)(g.inc >> 64), (unsigned long long)(uint64_t)g.inc);
#pragma unroll
        for (int k = 0; k < E::S; k += 2)
            out[2 + k / 2] = make_ulonglong2((unsigned long long)__double_as_longlong(s[k]),
                                             (unsigned long long)__double_as_longlong(s[k + 1]));
        out[2 + E::S / 2] = make_ulonglong2((unsigned long long)(uint32_t)elapsed |
                                                ((unsigned long long)a.flags[f] << 32), 0ULL);
#pragma unroll
        for (int c = 2 + E::S / 2 + 1; c < C; c++) out[c] = make_ulonglong2(0ULL, 0ULL);
        store_row<E::D>(q.end_obs, b, o);
    }
}

// reset(options={"low", "high"}) of env i (reset_kernel): state, TimeLimit counter, flags and, if obs is given, the
// observation row.  References as in lunar_reset_env.
template <int KIND>
__device__ __forceinline__ void reset_env_bounded(double *const &state, int32_t *const &elapsed, uint8_t *const &flags,
                                                  uint64_t *const &rng, float *const &obs, const int64_t &n, int64_t i,
                                                  const double &lo, const double &hi) {
    using E = bgym::Env<KIND>;
    double s[E::S];
    float o[E::D];
    bgym::Pcg64 g = bgym::pcg64_load(rng + 4 * i);
    E::reset(s, g, lo, hi, o);
    bgym::pcg64_store(rng + 4 * i, g);
#pragma unroll
    for (int k = 0; k < E::S; k++) state[k * n + i] = s[k];
    elapsed[i] = 0;
    flags[i] = 0;
    if (obs) store_row<E::D>(obs, i, o);
}

// ---- Box2D tasks -----------------------------------------------------------------------------------------------
// A step is up to three passes over a launch range [first, first + count): the step pass over every env, the TOI
// pass over the envs the step pass parked (toi_list), and the reset pass over the envs whose episode ended
// (reset_list).  With the lists null, the step pass does everything inline.

// side buffer of a parked env ([kToiMidWords][n] SoA): the sweep starts of the 3 bodies + env_pre's intermediates
constexpr int kToiMidWords = 20;   // LunarLander uses 13, BipedalWalker 15

__device__ __forceinline__ void lunar_store_mid(const StepArgs &a, int64_t i, const lunar::World &W, const lunar::Mid &mid) {
    uint32_t *m = a.toi_mid + i;
    for (int b = 0; b < lunar::NB; b++) {
        m[(int64_t)(3 * b + 0) * a.n] = __float_as_uint(W.b[b].c0.x);
        m[(int64_t)(3 * b + 1) * a.n] = __float_as_uint(W.b[b].c0.y);
        m[(int64_t)(3 * b + 2) * a.n] = __float_as_uint(W.b[b].a0);
    }
    const unsigned long long mc = (unsigned long long)__double_as_longlong(mid.main_cost);
    const unsigned long long sc = (unsigned long long)__double_as_longlong(mid.side_cost);
    m[(int64_t)9 * a.n] = (uint32_t)mc; m[(int64_t)10 * a.n] = (uint32_t)(mc >> 32);
    m[(int64_t)11 * a.n] = (uint32_t)sc; m[(int64_t)12 * a.n] = (uint32_t)(sc >> 32);
}

__device__ __forceinline__ void lunar_load_mid(const StepArgs &a, int64_t i, lunar::World &W, lunar::Mid &mid) {
    const uint32_t *m = a.toi_mid + i;
    for (int b = 0; b < lunar::NB; b++) {
        W.b[b].c0.x = __uint_as_float(m[(int64_t)(3 * b + 0) * a.n]);
        W.b[b].c0.y = __uint_as_float(m[(int64_t)(3 * b + 1) * a.n]);
        W.b[b].a0 = __uint_as_float(m[(int64_t)(3 * b + 2) * a.n]);
    }
    mid.main_cost = __longlong_as_double((long long)(((unsigned long long)m[(int64_t)10 * a.n] << 32) | m[(int64_t)9 * a.n]));
    mid.side_cost = __longlong_as_double((long long)(((unsigned long long)m[(int64_t)12 * a.n] << 32) | m[(int64_t)11 * a.n]));
    mid.awake = true;   // only awake islands are parked
}

// reset() of env i in place: record, RNG and TimeLimit counter; the new observation goes to obs.  The arrays and n
// are taken by reference, so that lunar_reset_list_kernel reads them from its parameter block where they are used;
// taken by value they are loaded up front, and the compiler allocates and schedules that kernel differently.
__device__ __forceinline__ void lunar_reset_env(uint32_t *const &rec, int32_t *const &elapsed, uint64_t *const &rng,
                                                const int64_t &n, int64_t i, const lunar::Opts &O, float (&obs)[8]) {
    lunar::World W;
    W.flags = rec[(int64_t)lunar::W_FLAGS * n + i] & b2l::kFlagsKept;  // the b2World object survives reset()
    W.wind_idx = O.wind ? (int32_t)rec[(int64_t)lunar::W_WIND * n + i] : 0;          // so do wind_idx / torque_idx
    W.torque_idx = O.wind ? (int32_t)rec[(int64_t)(lunar::W_WIND + 1) * n + i] : 0;
    bgym::Pcg64 g = bgym::pcg64_load(rng + 4 * i);
    lunar::env_reset(W, g, O, obs);
    lunar::store_world(W, rec, n, i, O.wind != 0);
    bgym::pcg64_store(rng + 4 * i, g);
    elapsed[i] = 0;
}

// everything after world.Step of LunarLander.step, then TimeLimit, outputs and the same-step autoreset
__device__ __noinline__ void lunar_finish(const StepArgs &a, int64_t i, int64_t j, lunar::World &W, bgym::Pcg64 &g,
                                          int32_t elapsed, const lunar::Mid &mid) {
    const lunar::Opts &O = a.lunar_opts;
    float obs[8];
    double reward;
    bool terminated;
    lunar::env_post(W, mid, obs, reward, terminated);
    elapsed += 1;                                                        // time_limit.py:51
    const bool truncated = (a.max_steps > 0) && (elapsed >= a.max_steps);
    store_scalars_all(a, i, reward, terminated ? 1 : 0, truncated ? 1 : 0);
    bool deferred = false;
    if ((terminated || truncated) && a.autoreset) {                      // sync_vector_env.py:152-156
        if (a.final_obs) store_row<8>(a.final_obs, i, obs);
        if (a.reset_list) {  // the new episode is drawn by the reset pass, in warps full of resetting envs
            a.reset_list[a.first + atomicAdd(a.reset_count, 1)] = (int32_t)j;
            deferred = true;
        } else {
            lunar::env_reset(W, g, O, obs);
            elapsed = 0;
        }
    }
    lunar::store_world(W, a.lunar_rec, a.n, i, O.wind != 0);
    bgym::pcg64_store(a.rng + 4 * i, g);
    a.elapsed[i] = elapsed;
    if (!deferred) store_obs_all<8>(a, i, obs);
}

// Step pass of env first + j (lunar_step_kernel; nothing for j past the range): the discrete solve, then either the env
// is parked for the TOI pass or its continuous collision is solved inline and the step finished.  The action is loaded
// under the range check and the check repeated before the work, as the kernel always has: folded into one branch,
// the integer-action kernels compile differently.
template <typename ActT, bool CONT>
__device__ __forceinline__ void lunar_step_env(const StepArgs &a, int64_t j) {
    const bool in_range = j < a.count;
    const int64_t i = a.first + j;
    long long act = 0;
    float ca0 = 0.0f, ca1 = 0.0f;
    bool valid = in_range;
    if (in_range) {
        if constexpr (CONT) {
            const float2 c = __ldg(reinterpret_cast<const float2 *>(a.actions) + i);   // Box(2) float32, lunar_lander.py:285-287
            ca0 = c.x; ca1 = c.y;
        } else {
            act = (long long)__ldg(reinterpret_cast<const ActT *>(a.actions) + i);
            valid = !(act < 0 || act > 3);   // lunar_lander.py:482-484
        }
    }
    if (!in_range) return;
    if (!valid) {
        atomicAdd(a.invalid, 1ULL);
        *reinterpret_cast<volatile unsigned long long *>(a.invalid_seen) = 1ULL;
        store_scalars_all(a, i, __longlong_as_double(0x7ff8000000000000LL), 0, 0);
        return;
    }
    const lunar::Opts &O = a.lunar_opts;
    lunar::World W;
    lunar::load_world(W, a.lunar_rec, a.n, i, O.wind != 0);
    bgym::Pcg64 g = bgym::pcg64_load(a.rng + 4 * i);
    const int32_t elapsed = a.elapsed[i];
    lunar::Mid mid;
    lunar::env_pre(W, g, O, (int)act, ca0, ca1, lunar::V(0.0f, 0.0f), mid, 0u, /*run_toi=*/false);
    if (mid.awake && b2l::toi_needed<lunar::Scene>(W)) {
        if (a.toi_list) {   // park the env for the TOI pass
            lunar::store_world(W, a.lunar_rec, a.n, i, O.wind != 0);
            bgym::pcg64_store(a.rng + 4 * i, g);
            lunar_store_mid(a, i, W, mid);
            a.toi_list[a.first + atomicAdd(a.toi_count, 1)] = (int32_t)j;
            return;
        }
        b2l::solve_toi<lunar::Scene>(W, (float)(1.0 / 50), true, 0u);
    }
    lunar_finish(a, i, j, W, g, elapsed, mid);
}

// TOI pass of entry idx of the parked list (lunar_toi_kernel); `live`: the lanes of the warp that run it together
__device__ __forceinline__ void lunar_toi_env(const StepArgs &a, int idx, unsigned live) {
    const lunar::Opts &O = a.lunar_opts;
    const int64_t j = a.toi_list[a.first + idx];
    const int64_t i = a.first + j;
    lunar::World W;
    lunar::load_world(W, a.lunar_rec, a.n, i, O.wind != 0);
    lunar::Mid mid;
    lunar_load_mid(a, i, W, mid);
    bgym::Pcg64 g = bgym::pcg64_load(a.rng + 4 * i);
    const int32_t elapsed = a.elapsed[i];
    b2l::solve_toi<lunar::Scene>(W, (float)(1.0 / 50), true, live);
    lunar_finish(a, i, j, W, g, elapsed, mid);
}

// reset pass of entry idx of the reset list (lunar_reset_list_kernel)
__device__ __forceinline__ void lunar_reset_list_env(const StepArgs &a, int idx) {
    const int64_t i = a.first + a.reset_list[a.first + idx];
    float obs[8];
    lunar_reset_env(a.lunar_rec, a.elapsed, a.rng, a.n, i, a.lunar_opts, obs);
    store_obs_all<8>(a, i, obs);
}

// side buffer of a parked walker env: the sweep starts of the bodies
__device__ __forceinline__ void walker_store_mid(const StepArgs &a, int64_t i, const walker::World &W) {
    uint32_t *m = a.toi_mid + i;
    for (int b = 0; b < walker::NB; b++) {
        m[(int64_t)(3 * b + 0) * a.n] = __float_as_uint(W.b[b].c0.x);
        m[(int64_t)(3 * b + 1) * a.n] = __float_as_uint(W.b[b].c0.y);
        m[(int64_t)(3 * b + 2) * a.n] = __float_as_uint(W.b[b].a0);
    }
}

__device__ __forceinline__ void walker_load_mid(const StepArgs &a, int64_t i, walker::World &W) {
    const uint32_t *m = a.toi_mid + i;
    for (int b = 0; b < walker::NB; b++) {
        W.b[b].c0.x = __uint_as_float(m[(int64_t)(3 * b + 0) * a.n]);
        W.b[b].c0.y = __uint_as_float(m[(int64_t)(3 * b + 1) * a.n]);
        W.b[b].a0 = __uint_as_float(m[(int64_t)(3 * b + 2) * a.n]);
    }
}

// reset() of env i in place: record (with the buffered 32-bit draw), RNG and TimeLimit counter; the new observation
// goes to obs.  References as in lunar_reset_env.
template <bool HC>
__device__ __forceinline__ void walker_reset_env(uint32_t *const &rec, int32_t *const &elapsed, uint64_t *const &rng,
                                                 const int64_t &n, int64_t i, float (&obs)[24]) {
    walker::World W;
    walker::Rng r;
    walker::bind_world(W, rec, n, i);
    W.flags = rec[(int64_t)walker::W_FLAGS * n + i] & b2l::kFlagsKept;  // the b2World object survives reset()
    r.has32 = rec[(int64_t)walker::W_RNG32 * n + i];
    r.val32 = rec[(int64_t)(walker::W_RNG32 + 1) * n + i];
    r.g = bgym::pcg64_load(rng + 4 * i);
    W.np = 0; W.p_lo = 0; W.p_hi = -1;
    walker::env_reset<HC>(W, r, obs);
    walker::store_world(W, rec, n, i, r, HC);
    bgym::pcg64_store(rng + 4 * i, r.g);
    elapsed[i] = 0;
}

// everything after world.Step of BipedalWalker.step, then TimeLimit, outputs and the same-step autoreset
template <bool HC>
__device__ __noinline__ void walker_finish(const StepArgs &a, int64_t i, int64_t j, walker::World &W, walker::Rng &rng,
                                           int32_t elapsed, const float (&action)[4]) {
    float obs[24];
    double reward;
    bool terminated;
    walker::env_post<HC>(W, action, false, obs, reward, terminated);
    elapsed += 1;                                                        // time_limit.py:51
    const bool truncated = (a.max_steps > 0) && (elapsed >= a.max_steps);
    store_scalars_all(a, i, reward, terminated ? 1 : 0, truncated ? 1 : 0);
    bool deferred = false;
    if ((terminated || truncated) && a.autoreset) {                      // sync_vector_env.py:152-156
        if (a.final_obs) store_row<24>(a.final_obs, i, obs);
        if (a.reset_list) {  // drawn by the reset pass (see lunar_finish)
            a.reset_list[a.first + atomicAdd(a.reset_count, 1)] = (int32_t)j;
            deferred = true;
        } else {
            rng.g = bgym::pcg64_load(a.rng + 4 * i);
            walker::env_reset<HC>(W, rng, obs);
            bgym::pcg64_store(a.rng + 4 * i, rng.g);
            elapsed = 0;
        }
    }
    walker::store_world(W, a.lunar_rec, a.n, i, rng, HC);
    a.elapsed[i] = elapsed;
    if (!deferred) store_obs_all<24>(a, i, obs);
}

// step pass of env first + j (walker_step_kernel), as lunar_step_env
template <bool HC>
__device__ __forceinline__ void walker_step_env(const StepArgs &a, int64_t j) {
    const int64_t i = a.first + j;
    const float4 av = __ldg(reinterpret_cast<const float4 *>(a.actions) + i);
    const float action[4] = {av.x, av.y, av.z, av.w};
    walker::World W;
    walker::Rng rng;
    walker::load_world(W, a.lunar_rec, a.n, i, rng, HC);
    const int32_t elapsed = a.elapsed[i];
    bool awake;
    walker::env_pre<HC>(W, action, walker::V(0.0f, 0.0f), awake, 0u, /*run_toi=*/false);
    if (awake && b2l::toi_needed<walker::SceneT<HC>>(W)) {
        if (a.toi_list) {   // park the env for the TOI pass: the record after the discrete solve + the sweep starts
            walker::store_world(W, a.lunar_rec, a.n, i, rng, HC);
            walker_store_mid(a, i, W);
            a.toi_list[a.first + atomicAdd(a.toi_count, 1)] = (int32_t)j;
            return;
        }
        b2l::solve_toi<walker::SceneT<HC>>(W, (float)(1.0 / 50), true, 0u);
    }
    walker_finish<HC>(a, i, j, W, rng, elapsed, action);
}

// TOI pass of entry idx of the parked list (walker_toi_kernel), as lunar_toi_env
template <bool HC>
__device__ __forceinline__ void walker_toi_env(const StepArgs &a, int idx, unsigned live) {
    const int64_t j = a.toi_list[a.first + idx];
    const int64_t i = a.first + j;
    const float4 av = __ldg(reinterpret_cast<const float4 *>(a.actions) + i);
    const float action[4] = {av.x, av.y, av.z, av.w};
    walker::World W;
    walker::Rng rng;
    walker::load_world(W, a.lunar_rec, a.n, i, rng, HC);
    walker_load_mid(a, i, W);
    // the window of obstacle boxes env_pre computed around the hull's position before the step
    if constexpr (HC) walker::poly_window(W, W.b[0].c0.x - 4.0f, W.b[0].c0.x + 4.0f, W.p_lo, W.p_hi);
    const int32_t elapsed = a.elapsed[i];
    b2l::solve_toi<walker::SceneT<HC>>(W, (float)(1.0 / 50), true, live);
    walker_finish<HC>(a, i, j, W, rng, elapsed, action);
}

// reset pass of entry idx of the reset list (walker_reset_list_kernel)
template <bool HC>
__device__ __forceinline__ void walker_reset_list_env(const StepArgs &a, int idx) {
    const int64_t i = a.first + a.reset_list[a.first + idx];
    float obs[24];
    walker_reset_env<HC>(a.lunar_rec, a.elapsed, a.rng, a.n, i, obs);
    store_obs_all<24>(a, i, obs);
}
