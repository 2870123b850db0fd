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
    // fused all-gather (multi-GPU): every result is ALSO stored into the same rows of the peers'
    // gather buffers over NVLink (peer-mapped pointers, slice offset already applied)
    // RecordEpisodeStatistics fused into the step (b200gym_set_episode_stats; nullptr = off): float32 return and
    // int32 length accumulators, infos["episode"]["r"/"l"] rows of finishing envs, ring of recent episodes
    float *ep_acc;
    int32_t *ep_len;
    float *ep_r;
    int32_t *ep_l;
    unsigned long long *ep_ring, *ep_counter;
    int32_t ep_ring_size;
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

// RecordEpisodeStatistics.step (gym/wrappers/record_episode_statistics.py:103-151) for env i, fused into the step
// kernels: `episode_returns += rewards` on a float32 array with float64 rewards (add in float64, round to float32),
// `episode_lengths += 1`; on terminated | truncated emit both, append to the ring (return_queue / length_queue),
// start over from zero.
template <typename I>
__device__ __forceinline__ void episode_account(const StepArgs &a, I i, double reward, bool done) {
    if (!a.ep_acc) return;
    const float ret = (float)((double)a.ep_acc[i] + reward);
    const int32_t len = a.ep_len[i] + 1;
    if (done) {
        a.ep_r[i] = ret;
        a.ep_l[i] = len;
        const unsigned long long slot = atomicAdd(a.ep_counter, 1ULL);
        if (a.ep_ring_size > 0)   // one 64-bit store per episode {length : return bits}: a slot never mixes two episodes
            a.ep_ring[slot % (unsigned long long)a.ep_ring_size] =
                ((unsigned long long)(uint32_t)len << 32) | (unsigned long long)__float_as_uint(ret);
        a.ep_acc[i] = 0.0f;
        a.ep_len[i] = 0;
    } else {
        a.ep_acc[i] = ret;
        a.ep_len[i] = len;
    }
}

// Where the results of env i go.  DirectSink: straight to the caller's arrays (and, when peers are mapped,
// to theirs) with per-thread stores.  The kernels that stage their outputs in shared memory have sinks of their own
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
template <int KIND, bool EP = true, typename Sink, typename I>
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
    if constexpr (EP) episode_account(a, i, reward, terminated || truncated);
    if (needs_reset) {
        if (a.final_obs) store_row<E::D>(a.final_obs, i, obs);           // info["final_observation"]
    } else {
        sink.template state<E::S>(i, s);
        sink.elapsed(i, elapsed);
        sink.template obs<E::D>(i, obs);
    }
    return needs_reset;
}

// Phase 2: the unseeded env.reset() of the autoreset (sync_vector_env.py:154) for env i, by
// whichever thread picked it off the CTA's compacted list.
template <int KIND, typename Sink, typename I>
__device__ __forceinline__ void reset_env(const StepArgs &a, const Sink &sink, I i) {
    using E = bgym::Env<KIND>;
    double s[E::S];
    float obs[E::D];
    bgym::Pcg64 g = bgym::pcg64_load(a.rng + 4 * (size_t)i);
    double lo, hi;
    E::default_bounds(lo, hi);
    E::reset(s, g, lo, hi, obs);
    bgym::pcg64_store(a.rng + 4 * (size_t)i, g);
    sink.template state<E::S>(i, s);
    sink.elapsed(i, 0);                                                  // time_limit.py:67
    sink.template obs<E::D>(i, obs);
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
    episode_account(a, i, reward, terminated || truncated);
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
    episode_account(a, i, reward, terminated || truncated);
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
