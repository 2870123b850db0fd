// b200gym.cu -- kernels + C ABI of the H100-native vectorised Gym engine.
//
// Hot path (reference: SyncVectorEnv.step_wait, gym/vector/sync_vector_env.py:135-169):
//   ONE kernel launch per vector step; one thread per environment instance;
//   Env.step + TimeLimit + same-step autoreset (with the env's own PCG64
//   stream) + observation/reward/flag emission fused.
//
// HBM layout (persistent, owned by the handle)
//   state   float64 [S][n]   SoA: lane i of a warp reads word k of env i -> 256 B
//                            contiguous per warp per word, fully coalesced
//   elapsed int32   [n]      TimeLimit._elapsed_steps
//   flags   uint8   [n]      bit0: "already terminated" (plain-Env mode only)
//   rng     uint64  [n][4]   numpy PCG64 {state_hi, state_lo, inc_hi, inc_lo}; AoS,
//                            touched only by lanes that reset
// I/O buffers are caller-owned (torch.cuda tensors): actions in; obs [n][D]
// float32, reward float64 [n], terminated/truncated uint8 [n], final_obs [n][D].
//
// Built for sm_90a only, with -fmad=false (see envs.cuh).
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <type_traits>

#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <string>

#include "../../include/b200gym.h"
#include "envs.cuh"
#include "lunar.cuh"
#include "walker.cuh"
#include "box2d_consts.h"
#include "per_env.cuh"
#include "rng.cuh"
#include "space_sample.cuh"
#include "subenv.cuh"

using namespace bgym;

// ---------------------------------------------------------------------------
// handle
// ---------------------------------------------------------------------------
struct b200gym {
    b200gym_config cfg;
    int64_t n = 0;
    int device = 0;
    int S = 0, D = 0, A = 0, NACT = 0;
    double *state = nullptr;
    int32_t *elapsed = nullptr;
    uint8_t *flags = nullptr;
    uint64_t *rng = nullptr;
    uint32_t *lunar_rec = nullptr;          // LunarLander / BipedalWalker: solver record, kWords 32-bit words per env, SoA
    bool is_lunar = false, is_walker = false;
    lunar::Opts lunar_opts{};
    unsigned long long *invalid = nullptr;  // sticky device counter
    unsigned long long *invalid_seen = nullptr;      // page-locked, device-mapped word: set to 1 by any kernel that meets an
    unsigned long long *invalid_seen_dev = nullptr;  // invalid action (host-visible WITHOUT a synchronisation); device alias
    int sm_count = 132;
    int occ[B200GYM_NUM_KINDS][3] = {};     // cached CTAs/SM of step_kernel_persistent per (kind, action width)
    int occ_bulk[B200GYM_NUM_KINDS][3] = {};  // ... of step_kernel_persistent_bulk per (kind, action width)
    int kernel_choice = -1;                 // -1: kernel B (bulk copies) where bulk_by_default picks it, else P;
                                            // 0: kernel A (one tile per CTA), 1: kernel P (resident grid, asynchronous
                                            // prefetch, deferred resets) where it applies, 2: kernel B where it applies
                                            // (else P); B200GYM_KERNEL=a|p|b overrides (l: the same as p)
    int box2d_defer = 1;                    // Box2D tasks: 1 = the autoresets of a step run in a last, compacted kernel
                                            // (B200GYM_BOX2D_DEFER=0: inline).  With the TOI kernel it takes reset() +
                                            // its embedded world step off the critical path of the envs that crash in a
                                            // TOI sub-step (H100 80GB HBM3 at 400 W, 2^16 envs, cold-L2 median:
                                            // LunarLander 1.82 -> 1.77 ms, BipedalWalker 9.16 -> 8.24 ms per step)
    int box2d_toi_defer = 1;                // Box2D tasks: 1 = envs with a possible TOI event finish in the compacted TOI kernel
                                            // (B200GYM_BOX2D_TOI_DEFER=0: SolveTOI inline in the step kernel)
    int32_t *toi_list = nullptr;            // [n] env offsets parked for the TOI kernel, per launch range
    int32_t *toi_count = nullptr;           // [kResetSlots]
    uint32_t *toi_mid = nullptr;            // [kToiMidWords][n] SoA side buffer of the parked envs
    int32_t *reset_list = nullptr;          // [n] env offsets to reset, filled per launch range
    int32_t *reset_count = nullptr;         // [kResetSlots] one counter per concurrently running launch range
    // fused all-gather over peer memory (b200gym_p2p_*)
    struct {
        int world = 0, rank = 0;
        unsigned char *base = nullptr;               // this rank's gather allocation (2 sets + flags)
        unsigned char *peer[B200GYM_MAX_PEERS + 1] = {};  // peer[r]: rank r's allocation mapped here (own = base)
        size_t set_bytes = 0, off_obs = 0, off_reward = 0, off_term = 0, off_trunc = 0, off_flags = 0, bytes = 0;
        unsigned long long step = 0;
        unsigned long long timeout_ns = 30ull * 1000000000ull;   // B200GYM_P2P_TIMEOUT_S overrides
        bool connected = false;
    } p2p;
    // host-I/O path (lazily created)
    b200gym_host_io hio{};
    b200gym_host_io dio{};  // device side: .actions in HBM; the result pointers are device aliases of hio's mapped buffers
    uint8_t *d_mask = nullptr;
    unsigned long long *h_invalid = nullptr;   // page-locked landing word of the invalid-action counter
    cudaEvent_t hevent = nullptr;
    unsigned long long **d_peer_flags = nullptr;
    unsigned int *p2p_done = nullptr;       // CTA counter of kernel G's fused step barrier
    bool p2p_barrier_fused = false;         // set by the last launch_step: the barrier ran in kernel G's tail
    int p2p_fuse = 0;                       // B200GYM_P2P_FUSE_BARRIER=1: the step barrier in kernel G's tail instead of the
                                            // 32-thread p2p_sync_kernel.  Correct (tests/test_gpu_multi.py runs it) but
                                            // slower than the separate launch: to vouch for its pushes a
                                            // CTA must wait for their COMPLETION (cp.async.bulk.wait_group 0: an NVLink
                                            // round trip per tile) instead of only for its tile to be read out of shared
                                            // memory, and that costs more residency than the kernel boundary + one tiny
                                            // launch save -- so the separate launch stays the default
    cudaStream_t hstream[2] = {nullptr, nullptr};
    bool host_ready = false;
    // env snapshots (lazily created)
    unsigned long long *snap_bad = nullptr;       // page-locked, device-mapped word: an out-of-range snapshot index was met
    unsigned long long *snap_bad_dev = nullptr;   // device alias
    unsigned char *snap_scratch = nullptr;        // b200gym_clone: n rows
    b200gym *from_batch = nullptr;                // b200gym_rollout_from, Box2D kinds: scratch batch (lazily created)
    float *norm_rows = nullptr;                   // normalised rollouts, Box2D kinds: n rows of D network inputs (lazily)
    // per-env wrapper chain (b200gym_subenv_set); the host-buffer path runs it inside its calls
    struct {
        bool on = false, out_f64 = false, episode = false;
        SubenvArgs args{};
        SubenvActions act{};                      // act.num == 0: no action stage
        double *final64 = nullptr;                // page-locked, mapped staging of the float64 final observations
        float *ep_r = nullptr;                    // ... of infos["final_info"][i]["episode"]["r"] / ["l"]
        int32_t *ep_l = nullptr;
        double *final64_dev = nullptr;            // their device aliases
        float *ep_r_dev = nullptr;
        int32_t *ep_l_dev = nullptr;
        // host-buffer path with a chain: the step and the chain run on these HBM copies of the outputs, which then go
        // to the mapped staging buffers as bulk copies (the terminal rows and episode fields of the finishing envs
        // are written there by the chain directly)
        float *obs = nullptr, *fin = nullptr;
        double *reward = nullptr;
        uint8_t *term = nullptr, *trunc = nullptr;
        float *out = nullptr;                     // [n][W] the chain's observations (reshaping chains)
    } sub;
    int obs_w = 0;                                // width of the host-buffer path's observation staging
    mutable std::string err;
};

static thread_local std::string g_create_err;

static int fail(const b200gym *h, const char *fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    if (h) h->err = buf;
    else g_create_err = buf;
    return 1;
}

#define CK(h, call)                                                                       \
    do {                                                                                  \
        cudaError_t e_ = (call);                                                          \
        if (e_ != cudaSuccess)                                                            \
            return fail(h, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
    } while (0)

static const int k_obs_dim[B200GYM_NUM_KINDS] = {4, 2, 2, 3, 6, 8, 24, 8, 24};
static const int k_act_dim[B200GYM_NUM_KINDS] = {0, 0, 1, 1, 0, 0, 4, 2, 4};
static const int k_nact[B200GYM_NUM_KINDS] = {2, 3, 0, 0, 3, 4, 0, 0, 0};
static const int k_state_dim[B200GYM_NUM_KINDS] = {4, 2, 2, 2, 4, 0, 0, 0, 0};

static bool kind_ok(int k) { return k >= 0 && k < B200GYM_NUM_KINDS; }

extern "C" int b200gym_obs_dim(int kind) { return kind_ok(kind) ? k_obs_dim[kind] : -1; }
extern "C" int b200gym_act_dim(int kind) { return kind_ok(kind) ? k_act_dim[kind] : -1; }
extern "C" int b200gym_num_actions(int kind) { return kind_ok(kind) ? k_nact[kind] : -1; }
extern "C" int b200gym_state_dim(int kind) { return kind_ok(kind) ? k_state_dim[kind] : -1; }
static int snap_row_bytes(int kind);
extern "C" int64_t b200gym_snapshot_row_bytes(int kind) { return kind_ok(kind) ? snap_row_bytes(kind) : -1; }
extern "C" int b200gym_version(void) { return B200GYM_VERSION; }
extern "C" const char *b200gym_last_error(const b200gym_t *h) {
    return h ? h->err.c_str() : g_create_err.c_str();
}
extern "C" int64_t b200gym_num_envs(const b200gym_t *h) { return h ? h->n : -1; }
extern "C" int b200gym_device(const b200gym_t *h) { return h ? h->device : -1; }

// ---------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------
constexpr int kThreads = 256;

// The sinks of the kernels that stage results in shared memory (the per-thread stores, DirectSinkT, are in
// per_env.cuh).  StagedSink, for kernel G: the outputs are staged, the persistent state goes straight back to HBM
struct StagedSink {
    float *s_obs;
    double *s_reward;
    uint8_t *s_term, *s_trunc;
    int64_t base;   // env index of row 0 of the tile
    const StepArgs &a;
    template <int D, typename I>
    __device__ __forceinline__ void obs(I i, const float (&v)[D]) const { store_row<D>(s_obs, (int)(i - base), v); }
    template <typename I>
    __device__ __forceinline__ void scalars(I i, double reward, uint8_t term, uint8_t trunc) const {
        const int r = (int)(i - base);
        s_reward[r] = reward; s_term[r] = term; s_trunc[r] = trunc;
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

// kernel B: every row that the tile's bulk stores cover is written into the tile's stage -- the new state and
// TimeLimit counter in place over the inputs, so that a row nobody writes (an invalid action) goes back to HBM
// unchanged.  The final observation is only handed back (`fin`, a register array
// of the calling thread): the kernel stores it after the warp has released the stage, so that no global store is
// outstanding at the warp's proxy fence
struct InPlaceSink {
    double *s_state;   // [S][kThreads]
    int32_t *s_elapsed;
    float *s_obs;
    double *s_reward;
    uint8_t *s_term, *s_trunc;
    uint32_t base;     // env index of row 0 of the tile
    float *fin;        // [D]
    template <int D, typename I>
    __device__ __forceinline__ void final_obs(I, const float (&v)[D]) const {
#pragma unroll
        for (int k = 0; k < D; k++) fin[k] = v[k];
    }
    template <int D, typename I>
    __device__ __forceinline__ void obs(I i, const float (&v)[D]) const { store_row<D>(s_obs, (int)(i - base), v); }
    template <typename I>
    __device__ __forceinline__ void scalars(I i, double reward, uint8_t term, uint8_t trunc) const {
        const int r = (int)(i - base);
        s_reward[r] = reward; s_term[r] = term; s_trunc[r] = trunc;
    }
    template <int S, typename I>
    __device__ __forceinline__ void state(I i, const double (&s)[S]) const {
        const int r = (int)(i - base);
#pragma unroll
        for (int k = 0; k < S; k++) s_state[k * kThreads + r] = s[k];
    }
    template <typename I>
    __device__ __forceinline__ void elapsed(I i, int32_t e) const { s_elapsed[(int)(i - base)] = e; }
};

// Tuning knobs (overridable at build time for A/B measurements).
// The per-env work is one long dependent float64 chain and the SMs are latency-bound, but occupancy is not the
// lever: at 32 registers (8 CTAs x 256 threads = 64 warps/SM) the hot loop spills the state across the division
// slow-path calls, and those local-memory round trips cost more than the extra warps hide.  6 CTAs/SM of 256
// threads leaves 40 registers a thread (64K registers per SM), which kernel P's loop fits without a spill.
#ifndef B200_MIN_CTAS
#define B200_MIN_CTAS 6
#endif
#ifndef B200_STAGES
#define B200_STAGES 2
#endif
template <int KIND>
struct Tuning {
    // Acrobot (RK4, ~70 live doubles) would spill heavily below 64 registers.  (The MountainCar kinds fit 32 registers
    // without a spill, which would make BASELINE's 2^18 envs one round of tiles instead of two; at 2^18 envs they are
    // latency-bound either way, so they keep the common budget.)
    static constexpr int kMinCtas = (KIND == B200GYM_ACROBOT) ? 3 : B200_MIN_CTAS;
    // kernel B (288 threads): 4 CTAs/SM = 32 compute warps and 56 registers a thread; the CTA's 3 stages of ~18 KB
    // (CartPole) leave 4 CTAs inside the SM's 228 KB of shared memory.  Acrobot: 2 CTAs, 113 registers
    static constexpr int kBulkMinCtas = (KIND == B200GYM_ACROBOT) ? 2 : 4;
};

// Why two phases: only ~1 env in 22 finishes per CartPole step, but then 77 % of the warps
// contain at least one finishing lane and would all walk the ~170-instruction PCG64 path
// (4 x 128-bit LCG steps) with 1-2 active lanes.  Instead finishing lanes push their env index
// onto a shared-memory list and, after one barrier, the first `count` threads of the CTA do
// the resets with full lanes: ~11 resets per 256-env tile = half a warp instead of 6 warps.

// --- kernel A: one thread per environment, inputs loaded straight from HBM -------------
// Used for small / ragged / unaligned batches and for the tail of kernel B.
template <int KIND, typename ActT>
__global__ void __launch_bounds__(kThreads, Tuning<KIND>::kMinCtas) step_kernel(const StepArgs a) {
    using E = Env<KIND>;
    __shared__ int reset_list[kThreads];
    __shared__ int reset_count;
    if (threadIdx.x == 0) reset_count = 0;
    __syncthreads();
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j < a.count) {
        const int64_t i = a.first + j;
        double s[E::S];
#pragma unroll
        for (int k = 0; k < E::S; k++) s[k] = a.state[k * a.n + i];
        const int32_t elapsed = a.elapsed[i];
        long long action_int = 0;
        float a0 = 0.0f;
        const ActT av = __ldg(reinterpret_cast<const ActT *>(a.actions) + i);
        decode_action<KIND>(av, action_int, a0);
        if (advance_env<KIND>(a, DirectSink{a}, i, s, elapsed, action_int, a0)) reset_list[atomicAdd(&reset_count, 1)] = threadIdx.x;
    }
    __syncthreads();
    const int cnt = reset_count;
    if ((int)threadIdx.x < cnt)
        reset_env<KIND>(a, DirectSink{a}, a.first + (int64_t)blockIdx.x * blockDim.x + reset_list[threadIdx.x]);
}

// --- rollout kernel: T steps per launch, one thread per environment ---------------------------------------------
// Thread i runs env i's T steps with the state and TimeLimit counter in registers (rollout_env); at every step a warp
// reads one coalesced action row and writes coalesced output rows of slice t.  A finishing env is reset inline, by
// its own lane, before its next step: the step kernels' deferred reset list does not apply
template <int KIND, typename ActT>
__global__ void __launch_bounds__(kThreads) rollout_kernel(const StepArgs a, const int32_t T, float *last_obs) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < a.n) rollout_env<KIND, ActT>(a, i, T, last_obs);
}

// ... with the actions drawn from the action space's stream as the kernel goes (rollout_sampled_env): the stream
// comes from the record (or the override) and the last CTA to take a ticket writes it back T * n draws later, as in
// space_sample_stream_kernel
template <int KIND>
__global__ void __launch_bounds__(kThreads) rollout_sampled_kernel(const StepArgs a, const int32_t T, float *last_obs,
                                                                   const RolloutDraws d, const SampleStream s) {
    __shared__ LcgJumpTable table;   // rows [0, jump_digits) of kLcgJump
    __shared__ Pcg64 start;
    const uint4 *src = reinterpret_cast<const uint4 *>(&kLcgJump);
    uint4 *dst = reinterpret_cast<uint4 *>(&table);
    for (int k = threadIdx.x; k < d.jump_digits * 32; k += kThreads) dst[k] = src[k];
    if (threadIdx.x == 0) start = sample_stream_start(s);
    __syncthreads();
    const Pcg64 g = start;
    // this CTA's read of the record has returned, so the last CTA to take a ticket writes after every read
    unsigned long long ticket = 0;
    if (threadIdx.x == 0) ticket = atomicAdd(reinterpret_cast<unsigned long long *>(s.record + 4), 1ULL);
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < a.n) rollout_sampled_env<KIND>(a, i, T, last_obs, d, g, table);
    if (threadIdx.x == 0 && ticket == gridDim.x - 1ULL) sample_stream_finish(s, g);
}

// ... with the actions computed by each env's linear policy from the observation of the step before
// (rollout_linear_env); SUMMARY: no per-step outputs, one episode summary per env
template <int KIND, bool SUMMARY>
__global__ void __launch_bounds__(kThreads) rollout_linear_kernel(const StepArgs a, const int32_t T, float *last_obs,
                                                                  const LinearPolicyArgs p) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < a.n) rollout_linear_env<KIND, SUMMARY>(a, i, T, last_obs, p);
}

// One step's actions of a Box2D linear-policy rollout, before that step's launches: env i's policy at its observation
// row obs[i] (K logits over D inputs, linear_logits), into actions[i] (int64 argmax_first if DISCRETE, else K float32).
// fold / init: the episode summary of b200gym_rollout_linear, folded from the step before's reward and flags
template <int K, int D, bool DISCRETE>
__global__ void __launch_bounds__(kThreads) linear_policy_kernel(const float *obs, void *actions,
                                                                 const LinearPolicyArgs p, const double *reward,
                                                                 const uint8_t *term, const uint8_t *trunc, int64_t n,
                                                                 int32_t t_prev, int act, int init) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (init) {
        p.returns[i] = 0.0;
        p.lengths[i] = 0;
        p.ended[i] = 0;
    } else if (t_prev >= 0 && !p.ended[i]) {   // step t_prev is the first episode end or before it
        p.returns[i] = p.returns[i] + reward[i];
        p.lengths[i] = t_prev + 1;
        p.ended[i] = (term[i] | trunc[i]) != 0;
    }
    if (!act) return;
    float o[D], w[K * D], b[K], z[K];
#pragma unroll
    for (int k = 0; k < D; k++) o[k] = obs[i * D + k];
#pragma unroll
    for (int k = 0; k < K * D; k++) w[k] = __ldg(p.weight + i * p.w_stride + k);
#pragma unroll
    for (int j = 0; j < K; j++) b[j] = __ldg(p.bias + i * p.b_stride + j);
    linear_logits<K, D>(w, b, o, z);
    if constexpr (DISCRETE) {
        static_cast<long long *>(actions)[i] = argmax_first<K>(z);
    } else {
#pragma unroll
        for (int j = 0; j < K; j++) static_cast<float *>(actions)[i * K + j] = z[j];
    }
}

// The CTA's shared copy of the `count` floats of one MLP policy shared by every env.  It is read from device memory at
// every launch, so a replayed CUDA graph uses the current contents of the parameters.  Every thread of the CTA calls it
__device__ __forceinline__ const float *mlp_stage(const float *params, int64_t count) {
    extern __shared__ float4 mlp_shared[];
    float *s = reinterpret_cast<float *>(mlp_shared);
    for (int64_t q = threadIdx.x; q < count; q += blockDim.x) s[q] = __ldg(params + q);
    __syncthreads();
    return s;
}

// ... with the actions computed by each env's MLP policy from the observation of the step before (rollout_mlp_env):
// PER_ENV, env i's row of parameters read from device memory at every step; otherwise one policy, staged in shared
// memory once per CTA.  SUMMARY: no per-step outputs, one episode summary per env.  ACT: the hidden layers' activation
// (mlp_act).  Held to 128 registers (two CTAs per SM), ptxas spills the per-env Pendulum kernels, so the per-env
// kernels ask for one CTA per SM instead
template <int KIND, bool SUMMARY, bool PER_ENV, int ACT>
__global__ void __launch_bounds__(kThreads, PER_ENV ? 1 : 2) rollout_mlp_kernel(const StepArgs a, const int32_t T, float *last_obs,
                                                               const MlpPolicyArgs p) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if constexpr (PER_ENV) {
        if (i < a.n) rollout_mlp_env<KIND, SUMMARY, true, ACT>(a, i, T, last_obs, p.params + i * p.stride, p);
    } else {
        using Src = MlpActions<KIND, SUMMARY, false, ACT>;
        const float *w = mlp_stage(p.params, mlp_param_count<Src::K, Src::D>(p.h1, p.h2));
        if (i < a.n) rollout_mlp_env<KIND, SUMMARY, false, ACT>(a, i, T, last_obs, w, p);
    }
}

// One step's actions of a Box2D MLP-policy rollout, before that step's launches: linear_policy_kernel with env i's
// MLP (mlp_outputs; PER_ENV and ACT as rollout_mlp_kernel) in place of its linear policy
template <int K, int D, bool DISCRETE, bool PER_ENV, int ACT>
__global__ void __launch_bounds__(kThreads) mlp_policy_kernel(const float *obs, void *actions, const MlpPolicyArgs p,
                                                              const double *reward, const uint8_t *term,
                                                              const uint8_t *trunc, int64_t n, int32_t t_prev, int act,
                                                              int init) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const float *w = nullptr;
    if (act) w = PER_ENV ? p.params + i * p.stride : mlp_stage(p.params, mlp_param_count<K, D>(p.h1, p.h2));
    if (i >= n) return;
    if (init) {
        p.returns[i] = 0.0;
        p.lengths[i] = 0;
        p.ended[i] = 0;
    } else if (t_prev >= 0 && !p.ended[i]) {   // step t_prev is the first episode end or before it
        p.returns[i] = p.returns[i] + reward[i];
        p.lengths[i] = t_prev + 1;
        p.ended[i] = (term[i] | trunc[i]) != 0;
    }
    if (!act) return;
    float o[D], z[K];
#pragma unroll
    for (int k = 0; k < D; k++) o[k] = obs[i * D + k];
    mlp_outputs<K, D, PER_ENV, ACT>(w, p.h1, p.h2, p.vec != 0, o, z);
    if constexpr (DISCRETE) {
        static_cast<long long *>(actions)[i] = argmax_first<K>(z);
    } else {
#pragma unroll
        for (int j = 0; j < K; j++) static_cast<float *>(actions)[i * K + j] = z[j];
    }
}

// ... with the actions computed by each env's MLP policy plus the caller's noise (rollout_mlp_noisy_env); PER_ENV, ACT
// and the launch bounds as rollout_mlp_kernel
template <int KIND, bool PER_ENV, int ACT>
__global__ void __launch_bounds__(kThreads, PER_ENV ? 1 : 2)
    rollout_mlp_noisy_kernel(const StepArgs a, const int32_t T, float *last_obs, const MlpNoisyArgs p) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if constexpr (PER_ENV) {
        if (i < a.n) rollout_mlp_noisy_env<KIND, true, ACT>(a, i, T, last_obs, p.mlp.params + i * p.mlp.stride, p);
    } else {
        using Src = MlpNoisyActions<KIND, false, ACT>;
        const float *w = mlp_stage(p.mlp.params, mlp_param_count<Src::K, Src::D>(p.mlp.h1, p.mlp.h2));
        if (i < a.n) rollout_mlp_noisy_env<KIND, false, ACT>(a, i, T, last_obs, w, p);
    }
}

// One step's actions of a Box2D noisy MLP-policy rollout: mlp_policy_kernel with the step's noise slice added to the
// outputs (noisy_outputs), which go to the step's outputs slice.  The launch passes p.noise and p.outputs at that
// step's slice.  No summary mode: reward, term, trunc, t_prev, act and init are the launcher's and unused here
template <int K, int D, bool DISCRETE, bool PER_ENV, int ACT>
__global__ void __launch_bounds__(kThreads) mlp_noisy_policy_kernel(const float *obs, void *actions,
                                                                    const MlpNoisyArgs p, const double *, const uint8_t *,
                                                                    const uint8_t *, int64_t n, int32_t, int, int) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const float *w = PER_ENV ? p.mlp.params + i * p.mlp.stride
                             : mlp_stage(p.mlp.params, mlp_param_count<K, D>(p.mlp.h1, p.mlp.h2));
    if (i >= n) return;
    float o[D], z[K], y[K];
#pragma unroll
    for (int k = 0; k < D; k++) o[k] = obs[i * D + k];
    mlp_outputs<K, D, PER_ENV, ACT>(w, p.mlp.h1, p.mlp.h2, p.mlp.vec != 0, o, z);
    noisy_outputs<K>(z, p.noise + i * K, p.outputs + i * K, y);
    if constexpr (DISCRETE) {
        static_cast<long long *>(actions)[i] = argmax_first<K>(y);
    } else {
#pragma unroll
        for (int j = 0; j < K; j++) static_cast<float *>(actions)[i * K + j] = y[j];
    }
}

// ... with the actions taken from each env's MLP policy through head HEAD, a b200gym_mlp_head (rollout_mlp_head_env);
// SUMMARY, PER_ENV, ACT and the launch bounds as rollout_mlp_kernel.  Classic Box kinds only
template <int KIND, bool SUMMARY, bool PER_ENV, int ACT, int HEAD>
__global__ void __launch_bounds__(kThreads, PER_ENV ? 1 : 2)
    rollout_mlp_head_kernel(const StepArgs a, const int32_t T, float *last_obs, const MlpHeadArgs p) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if constexpr (PER_ENV) {
        if (i < a.n)
            rollout_mlp_head_env<KIND, SUMMARY, true, ACT, HEAD>(a, i, T, last_obs, p.mlp.params + i * p.mlp.stride, p);
    } else {
        using Src = MlpHeadActions<KIND, SUMMARY, false, ACT, HEAD>;
        const float *w = mlp_stage(p.mlp.params, mlp_param_count<Src::K, Src::D>(p.mlp.h1, p.mlp.h2));
        if (i < a.n) rollout_mlp_head_env<KIND, SUMMARY, false, ACT, HEAD>(a, i, T, last_obs, w, p);
    }
}

// ... with the caller's noise going into head HEAD (rollout_mlp_noisy_head_env); PER_ENV, ACT and the launch bounds as
// rollout_mlp_kernel.  Classic Box kinds only
template <int KIND, bool PER_ENV, int ACT, int HEAD>
__global__ void __launch_bounds__(kThreads, PER_ENV ? 1 : 2)
    rollout_mlp_noisy_head_kernel(const StepArgs a, const int32_t T, float *last_obs, const MlpHeadArgs p) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if constexpr (PER_ENV) {
        if (i < a.n)
            rollout_mlp_noisy_head_env<KIND, true, ACT, HEAD>(a, i, T, last_obs, p.mlp.params + i * p.mlp.stride, p);
    } else {
        using Src = MlpNoisyHeadActions<KIND, false, ACT, HEAD>;
        const float *w = mlp_stage(p.mlp.params, mlp_param_count<Src::K, Src::D>(p.mlp.h1, p.mlp.h2));
        if (i < a.n) rollout_mlp_noisy_head_env<KIND, false, ACT, HEAD>(a, i, T, last_obs, w, p);
    }
}

// One step's actions of a Box2D MLP-policy rollout through head HEAD: mlp_policy_kernel for a Box kind with the K
// outputs going through the deterministic head (head_action) into the A actions
template <int K, int D, bool PER_ENV, int ACT, int HEAD>
__global__ void __launch_bounds__(kThreads) mlp_head_policy_kernel(const float *obs, void *actions, const MlpHeadArgs p,
                                                                   const double *reward, const uint8_t *term,
                                                                   const uint8_t *trunc, int64_t n, int32_t t_prev,
                                                                   int act, int init) {
    constexpr int A = HEAD == B200GYM_HEAD_TANH_NORMAL ? K / 2 : K;
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const float *w = nullptr;
    if (act)
        w = PER_ENV ? p.mlp.params + i * p.mlp.stride
                    : mlp_stage(p.mlp.params, mlp_param_count<K, D>(p.mlp.h1, p.mlp.h2));
    if (i >= n) return;
    if (init) {
        p.mlp.returns[i] = 0.0;
        p.mlp.lengths[i] = 0;
        p.mlp.ended[i] = 0;
    } else if (t_prev >= 0 && !p.mlp.ended[i]) {   // step t_prev is the first episode end or before it
        p.mlp.returns[i] = p.mlp.returns[i] + reward[i];
        p.mlp.lengths[i] = t_prev + 1;
        p.mlp.ended[i] = (term[i] | trunc[i]) != 0;
    }
    if (!act) return;
    float o[D], z[K], e[A] = {}, y[A];
#pragma unroll
    for (int k = 0; k < D; k++) o[k] = obs[i * D + k];
    mlp_outputs<K, D, PER_ENV, ACT>(w, p.mlp.h1, p.mlp.h2, p.mlp.vec != 0, o, z);
    head_action<HEAD, false>(z, e, p.bounds, y);
#pragma unroll
    for (int j = 0; j < A; j++) static_cast<float *>(actions)[i * A + j] = y[j];
}

// One step's actions of a Box2D noisy MLP-policy rollout through head HEAD: mlp_head_policy_kernel with the step's
// noise slice going into the head and the outputs to the step's outputs slice (the launch passes p.noise and p.outputs
// at that step's slice).  No summary mode: reward, term, trunc, t_prev, act and init are the launcher's and unused here
template <int K, int D, bool PER_ENV, int ACT, int HEAD>
__global__ void __launch_bounds__(kThreads) mlp_noisy_head_policy_kernel(const float *obs, void *actions,
                                                                         const MlpHeadArgs p, const double *,
                                                                         const uint8_t *, const uint8_t *, int64_t n,
                                                                         int32_t, int, int) {
    constexpr int A = HEAD == B200GYM_HEAD_TANH_NORMAL ? K / 2 : K;
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const float *w = PER_ENV ? p.mlp.params + i * p.mlp.stride
                             : mlp_stage(p.mlp.params, mlp_param_count<K, D>(p.mlp.h1, p.mlp.h2));
    if (i >= n) return;
    float o[D], z[K], e[A], y[A];
#pragma unroll
    for (int k = 0; k < D; k++) o[k] = obs[i * D + k];
    mlp_outputs<K, D, PER_ENV, ACT>(w, p.mlp.h1, p.mlp.h2, p.mlp.vec != 0, o, z);
#pragma unroll
    for (int k = 0; k < A; k++) e[k] = load_once(p.noise + i * A + k);
#pragma unroll
    for (int k = 0; k < K; k++) store_once(p.outputs + i * K + k, z[k]);
    head_action<HEAD, true>(z, e, p.bounds, y);
#pragma unroll
    for (int j = 0; j < A; j++) static_cast<float *>(actions)[i * A + j] = y[j];
}

// The CTA's shared copies of two nets, mlp_stage's for each: the `na` floats at a, then, from the next 16-byte boundary,
// the `nc` floats at c.  Returns the copy of c; the copy of a is at the start of the dynamic shared memory
__device__ __forceinline__ const float *mlp_stage_pair(const float *a, int64_t na, const float *c, int64_t nc) {
    extern __shared__ float4 mlp_shared[];
    float *s = reinterpret_cast<float *>(mlp_shared), *sc = s + (na + 3) / 4 * 4;
    for (int64_t q = threadIdx.x; q < na; q += blockDim.x) s[q] = __ldg(a + q);
    for (int64_t q = threadIdx.x; q < nc; q += blockDim.x) sc[q] = __ldg(c + q);
    __syncthreads();
    return sc;
}

// ... with the noisy actor's actions and the critic's values (rollout_actor_critic_env).  Both nets are shared by every
// env and staged in shared memory once per CTA, the actor first; launch bounds as the shared-policy noisy kernels
template <int KIND, int ACT>
__global__ void __launch_bounds__(kThreads, 2)
    rollout_actor_critic_kernel(const StepArgs a, const int32_t T, float *last_obs, const ActorCriticArgs p) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    using Src = MlpNoisyActions<KIND, false, ACT>;
    const int h1 = p.actor.mlp.h1, h2 = p.actor.mlp.h2;
    const float *wc = mlp_stage_pair(p.actor.mlp.params, mlp_param_count<Src::K, Src::D>(h1, h2), p.critic,
                                     mlp_param_count<1, Src::D>(h1, h2));
    extern __shared__ float4 mlp_shared[];
    if (i < a.n) rollout_actor_critic_env<KIND, ACT>(a, i, T, last_obs, reinterpret_cast<const float *>(mlp_shared),
                                                     wc, p);
}

// The advantages of a b200gym_rollout_actor_critic call, one thread per env (gae_env), after the rollout: a launch of
// its own for every kind, so the rollout kernel keeps its registers and the Box2D path shares it
__global__ void __launch_bounds__(kThreads) gae_kernel(const double *reward, const uint8_t *term, const uint8_t *trunc,
                                                       const float *values, float *adv, int64_t n, int32_t T, float g,
                                                       float gl) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) gae_env(i, n, T, g, gl, reward, term, trunc, values, adv);
}

// The CTA's shared copies of an observation normaliser's mean[D] and sd[D] = norm_sd(var[D], eps), computed by the
// first D threads; read from device memory at every launch, so a replayed CUDA graph uses the current statistics.  The
// caller's next __syncthreads (the parameters' staging) publishes them
template <int D>
__device__ __forceinline__ void norm_stage(const ObsNormArgs &q, double (&mean)[D], double (&sd)[D]) {
    if (threadIdx.x < D) {
        mean[threadIdx.x] = q.mean[threadIdx.x];
        sd[threadIdx.x] = norm_sd(q.var[threadIdx.x], q.eps);
    }
}

// rollout_mlp_noisy_kernel's shared-policy path with normalised inputs (rollout_mlp_noisy_norm_env); launch bounds as
// the shared-policy noisy kernels
template <int KIND, int ACT>
__global__ void __launch_bounds__(kThreads, 2)
    rollout_mlp_noisy_norm_kernel(const StepArgs a, const int32_t T, float *last_obs, const MlpNoisyArgs p,
                                  const ObsNormArgs q) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    using Src = MlpNoisyActions<KIND, false, ACT>;
    __shared__ double mean[Src::D], sd[Src::D];
    norm_stage<Src::D>(q, mean, sd);
    const float *w = mlp_stage(p.mlp.params, mlp_param_count<Src::K, Src::D>(p.mlp.h1, p.mlp.h2));
    if (i < a.n) rollout_mlp_noisy_norm_env<KIND, ACT>(a, i, T, last_obs, w, p, mean, sd, q.clip);
}

// rollout_actor_critic_kernel with normalised inputs for both nets (rollout_actor_critic_norm_env)
template <int KIND, int ACT>
__global__ void __launch_bounds__(kThreads, 2)
    rollout_actor_critic_norm_kernel(const StepArgs a, const int32_t T, float *last_obs, const ActorCriticArgs p,
                                     const ObsNormArgs q) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    using Src = MlpNoisyActions<KIND, false, ACT>;
    __shared__ double mean[Src::D], sd[Src::D];
    norm_stage<Src::D>(q, mean, sd);
    const int h1 = p.actor.mlp.h1, h2 = p.actor.mlp.h2;
    const float *wc = mlp_stage_pair(p.actor.mlp.params, mlp_param_count<Src::K, Src::D>(h1, h2), p.critic,
                                     mlp_param_count<1, Src::D>(h1, h2));
    extern __shared__ float4 mlp_shared[];
    if (i < a.n)
        rollout_actor_critic_norm_env<KIND, ACT>(a, i, T, last_obs, reinterpret_cast<const float *>(mlp_shared), wc, p,
                                                 mean, sd, q.clip);
}

// gae_kernel with the rewards scaled by the return statistics (gae_scaled_env): sd = norm_sd(ret_var[0], eps), read
// at every launch
__global__ void __launch_bounds__(kThreads) gae_scaled_kernel(const double *reward, const uint8_t *term,
                                                              const uint8_t *trunc, const float *values, float *adv,
                                                              int64_t n, int32_t T, float g, float gl,
                                                              const double *ret_var, double eps, float clip) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) gae_scaled_env(i, n, T, g, gl, norm_sd(__ldg(ret_var), eps), clip, reward, term, trunc, values, adv);
}

// rollout_linear_kernel with normalised inputs and, in summary mode, the observation moments (rollout_linear_norm_env).
// q.mean null: raw inputs; m.sum null: no moments.  Both branches are the same for every thread of the launch
template <int KIND, bool SUMMARY>
__global__ void __launch_bounds__(kThreads)
    rollout_linear_norm_kernel(const StepArgs a, const int32_t T, float *last_obs, const LinearPolicyArgs p,
                               const ObsNormArgs q, const ObsMomentArgs m) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    constexpr int D = bgym::Env<KIND>::D;
    __shared__ double mean[D], sd[D];
    if (q.mean) norm_stage<D>(q, mean, sd);
    __syncthreads();
    if (i < a.n) rollout_linear_norm_env<KIND, SUMMARY>(a, i, T, last_obs, p, q.mean ? mean : nullptr, sd, q.clip, m);
}

// rollout_mlp_kernel with normalised inputs and the observation moments (rollout_mlp_norm_env); q and m as
// rollout_linear_norm_kernel's, PER_ENV, ACT and the launch bounds as rollout_mlp_kernel's
template <int KIND, bool SUMMARY, bool PER_ENV, int ACT>
__global__ void __launch_bounds__(kThreads, PER_ENV ? 1 : 2)
    rollout_mlp_norm_kernel(const StepArgs a, const int32_t T, float *last_obs, const MlpPolicyArgs p,
                            const ObsNormArgs q, const ObsMomentArgs m) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    using Src = MlpActions<KIND, SUMMARY, PER_ENV, ACT>;
    __shared__ double mean[Src::D], sd[Src::D];
    if (q.mean) norm_stage<Src::D>(q, mean, sd);
    const double *mu = q.mean ? mean : nullptr;
    if constexpr (PER_ENV) {
        __syncthreads();
        if (i < a.n)
            rollout_mlp_norm_env<KIND, SUMMARY, true, ACT>(a, i, T, last_obs, p.params + i * p.stride, p, mu, sd, q.clip,
                                                           m);
    } else {
        const float *w = mlp_stage(p.params, mlp_param_count<Src::K, Src::D>(p.h1, p.h2));
        if (i < a.n) rollout_mlp_norm_env<KIND, SUMMARY, false, ACT>(a, i, T, last_obs, w, p, mu, sd, q.clip, m);
    }
}

// The observation moments of a Box2D summary-mode rollout, one step: env i adds its raw input row o[i] of step t
// (moments_fold's arithmetic) where step t is its first episode's end or before it.  Launched before step t's policy
// launch, which folds step t - 1 into the summary, so that is: t = 0 (onto +0.0), or neither the summary's `ended`
// (folded up to step t - 2) nor step t - 1's flags set
__global__ void __launch_bounds__(kThreads) obs_moments_kernel(const float *o, const uint8_t *ended,
                                                               const uint8_t *term, const uint8_t *trunc, int64_t n,
                                                               int D, int32_t t, const ObsMomentArgs m) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || (t > 0 && (ended[i] | term[i] | trunc[i]))) return;
    for (int k = 0; k < D; k++) {
        const int64_t e = i * D + k;
        const double v = (double)o[e];
        m.sum[e] = (t == 0 ? 0.0 : m.sum[e]) + v;
        m.sumsq[e] = (t == 0 ? 0.0 : m.sumsq[e]) + v * v;
    }
}

// --- asynchronous-copy helpers (sm_90a PTX) --------------------------------------------------------
namespace acp {

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// per-thread LDGSTS: global -> shared without a register in between (SASS LDGSTS)
template <int BYTES>
__device__ __forceinline__ void ld_async(void *smem_dst, const void *gmem_src) {
    static_assert(BYTES == 4 || BYTES == 8 || BYTES == 16, "cp.async moves 4, 8 or 16 bytes");
    if constexpr (BYTES == 16)
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src) : "memory");
    else
        asm volatile("cp.async.ca.shared.global [%0], [%1], %2;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src), "n"(BYTES) : "memory");
}
__device__ __forceinline__ void ld_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void ld_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// bulk (TMA, SASS UBLKCP) shared -> global store of a contiguous block; works on peer-mapped addresses
__device__ __forceinline__ void st_bulk(void *gmem_dst, const void *smem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gmem_dst), "r"(smem_u32(smem_src)),
                 "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void st_bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void st_bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// ... until the bulk copies of this thread are COMPLETE (their writes performed), not just their source read
__device__ __forceinline__ void st_bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
// generic-proxy writes to shared memory -> visible to the async proxy that executes the bulk copy
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// mbarrier in shared memory: `count` arrivals plus the transaction bytes announced by expect_tx complete a phase
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
// the initialised barriers -> visible to the async proxy (the bulk copies complete transactions on them)
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// until the phase of parity `parity` has completed
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    uint32_t ok;
    do {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok)
                     : "r"(smem_u32(bar)), "r"(parity)
                     : "memory");
    } while (!ok);
}
// bulk (TMA, SASS UBLKCP) global -> shared load of a contiguous block; its bytes complete on `bar`
__device__ __forceinline__ void ld_bulk(void *smem_dst, const void *gmem_src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

}  // namespace acp

__device__ __forceinline__ unsigned long long global_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// --- kernel P: persistent CTAs, per-thread asynchronous prefetch, CTA-deferred resets ---------------
// Kernel A is latency-bound: every warp issues its six loads, waits a cold HBM round trip, runs a ~330
// instruction float64 chain, stores and leaves; while it computes it has no load in flight, so the SM never
// holds the outstanding reads that Little's law asks for (3.35 TB/s x a loaded latency of the order of a
// microsecond, over 132 SMs: tens of KB per SM).  Here a resident grid (SMs x occupancy)
// walks the tiles; each THREAD copies the inputs of its env in the next tile (S state words, TimeLimit counter,
// action) into its own shared-memory slots with cp.async (LDGSTS: no registers, no barrier -- a thread only ever
// reads back what it wrote itself) while it advances the current tile, so loads stay in flight through the whole
// kernel.  Warps never meet at a barrier inside the loop: finishing envs go onto one CTA-wide list that is
// drained ONCE, with full lanes, after the loop (a warp where many lanes finish at once -- synchronised
// TimeLimit truncation -- resets inline instead, which is then equally dense).
constexpr int kResetCap = 1024;   // entries of the CTA's deferred-reset list; overflow resets inline

template <int KIND, typename ActT>
struct PrefetchLayout {
    using E = Env<KIND>;
    static constexpr int kActPerEnv = E::A == 0 ? 1 : E::A;
    static constexpr int kActBytes = kActPerEnv * (int)sizeof(ActT);
    static constexpr bool kActAsync = kActBytes == 4 || kActBytes == 8 || kActBytes == 16;
    static constexpr int kStateOff = 0;                                   // [S][256] float64
    static constexpr int kActOff = E::S * kThreads * 8;                   // [256] action (if async)
    static constexpr int kElapsedOff = kActOff + (kActAsync ? kThreads * kActBytes : 0);   // [256] int32
    static constexpr int kBytes = kElapsedOff + kThreads * 4;
};

// Single-GPU step of a handle of fewer than 2^30 envs (launch_step_typed checks): 32-bit env indices (one IMAD.WIDE
// per address instead of a 64-bit add chain) and no per-peer store loops.
template <int KIND, typename ActT>
__global__ void __launch_bounds__(kThreads, Tuning<KIND>::kMinCtas) step_kernel_persistent(const StepArgs a, const int num_tiles) {
    using E = Env<KIND>;
    using L = PrefetchLayout<KIND, ActT>;
    using Idx = uint32_t;
    // one stage of per-thread input slots holds the next tile in flight: a thread moves its slot into registers
    // before it refills it
    __shared__ __align__(16) unsigned char in_mem[L::kBytes];
    __shared__ int reset_list[kResetCap];
    __shared__ int reset_count;
    const int tid = threadIdx.x;
    if (tid == 0) reset_count = 0;
    __syncthreads();

    const ActT *actions = reinterpret_cast<const ActT *>(a.actions);
    const DirectSinkT<false> sink{a};
    const Idx first = (Idx)a.first, count = (Idx)a.count;

    auto prefetch = [&](int tile) {
        double *s_state = reinterpret_cast<double *>(in_mem + L::kStateOff);
        int32_t *s_elapsed = reinterpret_cast<int32_t *>(in_mem + L::kElapsedOff);
        const Idx j = (Idx)tile * kThreads + tid;
        if (tile < num_tiles && j < count) {
            const Idx i = first + j;
#pragma unroll
            for (int k = 0; k < E::S; k++) acp::ld_async<8>(s_state + k * kThreads + tid, a.state + k * a.n + i);
            acp::ld_async<4>(s_elapsed + tid, a.elapsed + i);
            if constexpr (L::kActAsync)
                acp::ld_async<L::kActBytes>(in_mem + L::kActOff + tid * L::kActBytes, actions + (size_t)i * L::kActPerEnv);
        }
        acp::ld_commit();
    };

    int tile = blockIdx.x;
    prefetch(tile);
    for (; tile < num_tiles; tile += gridDim.x) {
        const Idx j = (Idx)tile * kThreads + tid;
        const bool in_range = j < count;
        const Idx i = first + j;
        ActT av{};
        if constexpr (!L::kActAsync) { if (in_range) av = __ldg(actions + (size_t)i * L::kActPerEnv); }
        acp::ld_wait_all();
        const double *s_state = reinterpret_cast<const double *>(in_mem + L::kStateOff);
        double s[E::S];
#pragma unroll
        for (int k = 0; k < E::S; k++) s[k] = s_state[k * kThreads + tid];
        const int32_t elapsed = reinterpret_cast<const int32_t *>(in_mem + L::kElapsedOff)[tid];
        if constexpr (L::kActAsync) av = *reinterpret_cast<const ActT *>(in_mem + L::kActOff + tid * L::kActBytes);
        // this thread's slots are in registers now: refill them with its env of the next round
        prefetch(tile + (int)gridDim.x);
        long long action_int = 0;
        float a0 = 0.0f;
        decode_action<KIND>(av, action_int, a0);
        bool need = false;
        if (in_range) need = advance_env<KIND>(a, sink, i, s, elapsed, action_int, a0);
        const unsigned m = __ballot_sync(0xffffffffu, need);
        if (m != 0u) {
            bool inline_reset = __popc(m) >= 12;          // dense enough: reset right here
            if (need && !inline_reset) {
                const int slot = atomicAdd(&reset_count, 1);
                if (slot < kResetCap) {
                    reset_list[slot] = (int)j;
                    // the drain after the loop starts with this env's 32-byte PCG64 record: have it in L2 by then
                    asm volatile("prefetch.global.L2 [%0];" ::"l"(a.rng + 4 * (size_t)i));
                } else inline_reset = true;               // list full (whole batch truncating at once)
            }
            if (need && inline_reset) reset_env<KIND>(a, sink, i);
        }
    }
    __syncthreads();
    const int cnt = min(reset_count, kResetCap);
    for (int q = tid; q < cnt; q += kThreads) reset_env<KIND>(a, sink, (Idx)(first + (Idx)reset_list[q]));
}

// --- kernel B: kernel P's resident grid with every HBM row moved by bulk copies -------------------------------
// In kernel P each compute warp is also its own memory engine: per tile it issues S + 2 per-thread cp.async and
// S + 5 per-thread stores, and when HBM is saturated those instructions queue behind each other in the LSU, so the
// arithmetic advances only as fast as memory accepts requests.  Here one extra warp (one elected thread) moves the
// tiles: a ring of kBulkStages stages per CTA, each filled by S + 2 bulk loads (state rows, TimeLimit counters,
// actions) that complete on the stage's `full` mbarrier.  The 8 compute warps read their env's inputs from the
// stage, write every result back INTO the stage (new state and counter in place, obs / reward / flags in the
// stage's output block: InPlaceSink), fence the writes to the async proxy and arrive on the stage's `done`
// mbarrier; the copy thread then pushes the whole tile out with S + 5 bulk stores and, once they have read the
// stage, refills it with the tile kBulkStages rounds ahead.  So the compute warps execute only shared-memory loads and
// stores on the common path.  Every finishing env is reset inside the stage, before the warp's `done` arrive, so a
// CTA is finished with a tile once its bulk stores have been issued.  The reset's one global load is the env's
// 32-byte PCG64 record.  Where the kind can tell from a tile's inputs which envs will finish (will_reset: CartPole),
// the record is requested into L2 as soon as the warp has read its inputs, so that it arrives while the float64 step
// runs.  An env that resets without having been predicted loads its record then; correctness never depends on the
// prediction.
// Whole tiles only, every row 16-byte aligned (launch_step_typed checks), 32-bit env indices.
constexpr int kBulkStages = 3;   // 2 stages at 5 CTAs/SM measured slower (DESIGN §4.1)

// Phase clocks of kernel B (-DB200_PHASE_CLOCKS, scripts/cartpole_phases.py; the default build compiles none of it).
// Lane 0 of every compute warp and the copy thread add clock() cycles per phase into g_phase_cycles; every CTA
// stamps %globaltimer at its start, when its last compute warp leaves the loop, and when its copy thread exits.
// b200gym_phase_clocks reads (and clears) both.
#ifdef B200_PHASE_CLOCKS
enum PhaseBucket {
    kPhFull, kPhAdvance, kPhRecord, kPhReset, kPhArrive, kPhComputeLoop, kPhComputeTiles,   // compute warps (lane 0)
    kPhDone, kPhStore, kPhWaitRead, kPhLoad, kPhFinalWait, kPhCopyLoop,                         // copy thread
    kPhBuckets
};
constexpr int kPhMaxCtas = 4096;
__device__ unsigned long long g_phase_cycles[kPhBuckets];
__device__ unsigned long long g_phase_ns[kPhMaxCtas][3];   // start, loop end, exit
// 32-bit clocks (differences are exact modulo 2^32) and per-warp sums in shared memory: the instrumented loop
// keeps no extra 64-bit registers live, so it runs with the registers of the default build
#define PH_CLOCK(t) const unsigned t = (unsigned)clock()
#define PH_DECL()                                                                              \
    __shared__ unsigned ph_s[kThreads / 32 + 1][kPhBuckets];                                  \
    __shared__ unsigned ph_zero;                                                               \
    for (int b_ = threadIdx.x; b_ < (kThreads / 32 + 1) * kPhBuckets; b_ += blockDim.x) (&ph_s[0][0])[b_] = 0u
#define PH_ACC(b, t0, t1) \
    do { if ((threadIdx.x & 31) == 0) ph_s[threadIdx.x >> 5][b] += (t1) - (t0); } while (0)
// an instruction that reads v, so that a clock read after it comes after v's load has completed
#define PH_USE(v) \
    do { if ((v) == 0ull) ph_zero = 1u; } while (0)
#define PH_FLUSH()                                                                             \
    do {                                                                                       \
        if (threadIdx.x < kPhBuckets) {                                                        \
            unsigned long long s_ = 0;                                                         \
            for (int w_ = 0; w_ < kThreads / 32 + 1; w_++) s_ += ph_s[w_][threadIdx.x];        \
            atomicAdd(&g_phase_cycles[threadIdx.x], s_);                                       \
        }                                                                                      \
    } while (0)
#define PH_STAMP(slot) \
    do { if (blockIdx.x < kPhMaxCtas) g_phase_ns[blockIdx.x][slot] = global_ns(); } while (0)
#define PH_STAMP_MAX(slot) \
    do { if (blockIdx.x < kPhMaxCtas) atomicMax(&g_phase_ns[blockIdx.x][slot], global_ns()); } while (0)

extern "C" int b200gym_phase_clocks(unsigned long long *cycles, unsigned long long *ns, int clear) {
    if (cudaMemcpyFromSymbol(cycles, g_phase_cycles, sizeof g_phase_cycles) != cudaSuccess) return 1;
    if (cudaMemcpyFromSymbol(ns, g_phase_ns, sizeof g_phase_ns) != cudaSuccess) return 1;
    if (clear) {
        static const unsigned long long zc[kPhBuckets] = {};
        static unsigned long long zn[kPhMaxCtas][3] = {};
        if (cudaMemcpyToSymbol(g_phase_cycles, zc, sizeof zc) != cudaSuccess) return 1;
        if (cudaMemcpyToSymbol(g_phase_ns, zn, sizeof zn) != cudaSuccess) return 1;
    }
    return 0;
}
#else
#define PH_CLOCK(t)
#define PH_DECL()
#define PH_ACC(b, t0, t1)
#define PH_USE(v)
#define PH_FLUSH()
#define PH_STAMP(slot)
#define PH_STAMP_MAX(slot)
#endif

template <int KIND, typename ActT>
struct BulkLayout {
    using E = Env<KIND>;
    static constexpr int kActPerEnv = E::A == 0 ? 1 : E::A;
    static constexpr int kStateOff = 0;                                       // [S][256] float64, in place
    static constexpr int kElapsedOff = E::S * kThreads * 8;                   // [256] int32, in place
    static constexpr int kActOff = kElapsedOff + kThreads * 4;                // [256][A] actions
    static constexpr int kObsOff = kActOff + kThreads * kActPerEnv * (int)sizeof(ActT);   // [256][D] float32
    static constexpr int kRewardOff = kObsOff + kThreads * E::D * 4;          // [256] float64
    static constexpr int kTermOff = kRewardOff + kThreads * 8;                // [256] uint8
    static constexpr int kTruncOff = kTermOff + kThreads;                     // [256] uint8
    static constexpr int kBytes = kTruncOff + kThreads;
    static constexpr uint32_t kLoadBytes = kObsOff;                           // the bulk loads fill [0, kObsOff)
    static_assert(kActOff % 16 == 0 && kObsOff % 16 == 0 && kBytes % 128 == 0, "bulk copies need 16-byte rows");
};

template <int KIND, typename ActT>
__global__ void __launch_bounds__(kThreads + 32, Tuning<KIND>::kBulkMinCtas)
    step_kernel_persistent_bulk(const StepArgs a, const int num_tiles) {
    using E = Env<KIND>;
    using L = BulkLayout<KIND, ActT>;
    extern __shared__ __align__(128) unsigned char stage_mem[];   // [kBulkStages][L::kBytes]
    // per stage: full = its inputs have landed, done = the compute warps are through with it
    __shared__ __align__(8) uint64_t full[kBulkStages], done[kBulkStages];
    const int tid = threadIdx.x;
    PH_DECL();
    if (tid == 0) {
        PH_STAMP(0);
        for (int q = 0; q < kBulkStages; q++) {
            acp::mbar_init(&full[q], 1);
            acp::mbar_init(&done[q], kThreads / 32);
        }
        acp::fence_mbar_init();
    }
    __syncthreads();
    const uint32_t first = (uint32_t)a.first, n = (uint32_t)a.n;

    if (tid >= kThreads) {
        if (tid == kThreads) {   // the copy thread
            auto load = [&](int tile, int q) {
                unsigned char *b = stage_mem + q * L::kBytes;
                const uint32_t i0 = first + (uint32_t)tile * kThreads;
                acp::mbar_arrive_expect_tx(&full[q], L::kLoadBytes);
#pragma unroll
                for (int k = 0; k < E::S; k++)
                    acp::ld_bulk(b + L::kStateOff + k * kThreads * 8, a.state + k * n + i0, kThreads * 8, &full[q]);
                acp::ld_bulk(b + L::kElapsedOff, a.elapsed + i0, kThreads * 4, &full[q]);
                acp::ld_bulk(b + L::kActOff, reinterpret_cast<const ActT *>(a.actions) + i0 * L::kActPerEnv,
                             L::kObsOff - L::kActOff, &full[q]);
            };
            auto store = [&](int tile, int q) {
                const unsigned char *b = stage_mem + q * L::kBytes;
                const uint32_t i0 = first + (uint32_t)tile * kThreads;
#pragma unroll
                for (int k = 0; k < E::S; k++) acp::st_bulk(a.state + k * n + i0, b + L::kStateOff + k * kThreads * 8, kThreads * 8);
                acp::st_bulk(a.elapsed + i0, b + L::kElapsedOff, kThreads * 4);
                acp::st_bulk(a.obs + i0 * E::D, b + L::kObsOff, kThreads * E::D * 4);
                acp::st_bulk(a.reward + i0, b + L::kRewardOff, kThreads * 8);
                acp::st_bulk(a.terminated + i0, b + L::kTermOff, kThreads);
                acp::st_bulk(a.truncated + i0, b + L::kTruncOff, kThreads);
                acp::st_bulk_commit();
            };
            int q = 0;
            for (int t = blockIdx.x; q < kBulkStages && t < num_tiles; t += gridDim.x) load(t, q++);
            q = 0;
            uint32_t parity = 0;
            PH_CLOCK(c_begin);
            for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
                PH_CLOCK(c0);
                acp::mbar_wait(&done[q], parity);
                PH_CLOCK(c1);
                store(tile, q);
                PH_CLOCK(c2);
                PH_ACC(kPhDone, c0, c1);
                PH_ACC(kPhStore, c1, c2);
                const int next = tile + kBulkStages * (int)gridDim.x;
                if (next < num_tiles) {
                    // the stage is free once the stores have READ it (a few hundred ns); waiting right away keeps
                    // kBulkStages - 1 tiles of loads ahead of the compute warps instead of kBulkStages - 2
                    acp::st_bulk_wait_read();
                    PH_CLOCK(c3);
                    load(next, q);
                    PH_CLOCK(c4);
                    PH_ACC(kPhWaitRead, c2, c3);
                    PH_ACC(kPhLoad, c3, c4);
                }
                if (++q == kBulkStages) { q = 0; parity ^= 1u; }
            }
            PH_CLOCK(c_end);
            acp::st_bulk_wait_read();    // the stages must outlive the stores that read them
            PH_CLOCK(c_drained);
            PH_ACC(kPhCopyLoop, c_begin, c_end);
            PH_ACC(kPhFinalWait, c_end, c_drained);
        }
    } else {
        const int lane = tid & 31;
        int q = 0;
        uint32_t parity = 0;
        PH_CLOCK(w_begin);
        for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
            PH_CLOCK(w0);
            unsigned char *b = stage_mem + q * L::kBytes;
            const uint32_t i = first + (uint32_t)tile * kThreads + tid;
            uint64_t *const rec = a.rng + 4 * (size_t)i;
            float fin[E::D];
            const InPlaceSink sink{reinterpret_cast<double *>(b + L::kStateOff), reinterpret_cast<int32_t *>(b + L::kElapsedOff),
                                   reinterpret_cast<float *>(b + L::kObsOff), reinterpret_cast<double *>(b + L::kRewardOff),
                                   b + L::kTermOff, b + L::kTruncOff, i - tid, fin};
            acp::mbar_wait(&full[q], parity);
            PH_CLOCK(w1);
            PH_ACC(kPhFull, w0, w1);
            double s[E::S];
#pragma unroll
            for (int k = 0; k < E::S; k++) s[k] = sink.s_state[k * kThreads + tid];
            const int32_t elapsed = sink.s_elapsed[tid];
            const ActT av = reinterpret_cast<const ActT *>(b + L::kActOff)[tid * L::kActPerEnv];
            long long action_int = 0;
            float a0 = 0.0f;
            decode_action<KIND>(av, action_int, a0);
            if (will_reset<KIND>(a, s, elapsed, action_int)) asm volatile("prefetch.global.L2 [%0];" ::"l"(rec));
            const bool need = advance_env<KIND>(a, sink, i, s, elapsed, action_int, a0);
            PH_CLOCK(w2);
            PH_ACC(kPhAdvance, w1, w2);
            // the reset through the stage; the record's write-back, like the final observation, waits until the
            // stage is released, so that no global store is outstanding at the proxy fence
            bgym::Pcg64 g;
            if (need) {
                g = bgym::pcg64_load(rec);
                PH_USE((uint64_t)g.state);
            }
            PH_CLOCK(w3);
            PH_ACC(kPhRecord, w2, w3);
            if (need) reset_env_from<KIND>(sink, i, g);
            PH_CLOCK(w4);
            PH_ACC(kPhReset, w3, w4);
            acp::fence_async_smem();
            __syncwarp();
            if (lane == 0) acp::mbar_arrive(&done[q]);
            if (need) {
                if (a.final_obs) store_row<E::D>(a.final_obs, i, fin);
                bgym::pcg64_store(rec, g);
            }
            PH_CLOCK(w5);
            PH_ACC(kPhArrive, w4, w5);
            PH_ACC(kPhComputeTiles, 0, 1);
            if (++q == kBulkStages) { q = 0; parity ^= 1u; }
        }
        PH_CLOCK(w_end);
        PH_ACC(kPhComputeLoop, w_begin, w_end);
        if (lane == 0) PH_STAMP_MAX(1);
    }
#ifdef B200_PHASE_CLOCKS
    __syncthreads();
    if (tid == 0) PH_STAMP(2);
    PH_FLUSH();
#endif
}

// --- kernel G: one tile per CTA, results staged in shared memory and pushed with bulk stores ---------
// The multi-GPU step (b200gym_step_p2p): every result must land in this rank's rows of EVERY rank's gather
// buffers.  Per-thread peer stores put 16-, 8- and 1-byte writes on NVLink; here the 256-env tile of
// (obs, reward, terminated, truncated) is assembled in shared memory (reset observations included) and warp w
// pushes it to destination w -- peer w, or this rank's own buffers -- as four bulk copies (cp.async.bulk
// shared -> global, SASS UBLKCP), so NVLink carries full-size write packets and the LSU carries none of it.
// Needs 16-byte aligned destination rows; ragged tails and unaligned shards use kernel A's per-thread stores.
template <int KIND, typename ActT>
__global__ void __launch_bounds__(kThreads, Tuning<KIND>::kMinCtas) step_kernel_gather(const StepArgs a) {
    using E = Env<KIND>;
    __shared__ __align__(128) float s_obs[kThreads * E::D];
    __shared__ __align__(16) double s_reward[kThreads];
    __shared__ __align__(16) uint8_t s_term[kThreads];
    __shared__ __align__(16) uint8_t s_trunc[kThreads];
    __shared__ int reset_list[kThreads];
    __shared__ int reset_count;
    if (threadIdx.x == 0) reset_count = 0;
    __syncthreads();
    const int64_t j0 = (int64_t)blockIdx.x * kThreads;      // full tiles only: no bound check
    const int64_t i0 = a.first + j0;
    const StagedSink sink{s_obs, s_reward, s_term, s_trunc, i0, a};
    {
        const int64_t i = i0 + threadIdx.x;
        double s[E::S];
#pragma unroll
        for (int k = 0; k < E::S; k++) s[k] = a.state[k * a.n + i];
        const int32_t elapsed = a.elapsed[i];
        long long action_int = 0;
        float a0 = 0.0f;
        const ActT av = __ldg(reinterpret_cast<const ActT *>(a.actions) + i);
        decode_action<KIND>(av, action_int, a0);
        if (advance_env<KIND>(a, sink, i, s, elapsed, action_int, a0)) reset_list[atomicAdd(&reset_count, 1)] = threadIdx.x;
    }
    __syncthreads();
    if ((int)threadIdx.x < reset_count) reset_env<KIND>(a, sink, i0 + reset_list[threadIdx.x]);
    acp::fence_async_smem();
    __syncthreads();
    const int warp = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0 && warp <= a.npeer) {
        float *obs = warp < a.npeer ? a.peer_obs[warp] : a.obs;
        double *reward = warp < a.npeer ? a.peer_reward[warp] : a.reward;
        uint8_t *term = warp < a.npeer ? a.peer_term[warp] : a.terminated;
        uint8_t *trunc = warp < a.npeer ? a.peer_trunc[warp] : a.truncated;
        acp::st_bulk(obs + i0 * E::D, s_obs, kThreads * E::D * 4);
        acp::st_bulk(reward + i0, s_reward, kThreads * 8);
        acp::st_bulk(term + i0, s_term, kThreads);
        acp::st_bulk(trunc + i0, s_trunc, kThreads);
        acp::st_bulk_commit();
        if (a.p2p_done) acp::st_bulk_wait_all();   // the step barrier below vouches for these writes
        else acp::st_bulk_wait_read();             // the tile must stay in shared memory until the copy engine has read it
    }
    if (a.p2p_done) {
        // the exchange's step barrier, fused: every CTA counts itself in once its pushes are complete; the last one
        // of this rank tells every peer "my rows of this step are in your buffers" and waits for theirs
        __syncthreads();
        __shared__ int is_last;
        if (threadIdx.x == 0) {
            __threadfence_system();
            const unsigned prev = atomicAdd(a.p2p_done, 1u);
            is_last = prev == gridDim.x - 1;
            if (is_last) *a.p2p_done = 0u;         // for the next launch (this one has no more increments coming)
        }
        __syncthreads();
        if (is_last && (int)threadIdx.x < a.p2p_world && (int)threadIdx.x != a.p2p_rank) {
            const int p = threadIdx.x;
            __threadfence_system();
            volatile unsigned long long *f = a.p2p_peer_flags[p] + a.p2p_rank;
            *f = a.p2p_step;
            const volatile unsigned long long *w = a.p2p_my_flags + p;
            const unsigned long long t0 = global_ns();
            while (*w < a.p2p_step) {
                if (global_ns() - t0 > a.p2p_timeout_ns) {
                    atomicExch(a.p2p_timed_out, p + 1);
                    break;
                }
            }
            __threadfence_system();
        }
    }
}

template <int KIND>
__global__ void __launch_bounds__(kThreads) reset_kernel(double *state, int32_t *elapsed, uint8_t *flags,
                                                         uint64_t *rng, const uint8_t *mask, float *obs,
                                                         int64_t n, double lo, double hi) {
    const int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    if (mask && !mask[i]) return;
    reset_env_bounded<KIND>(state, elapsed, flags, rng, obs, n, i, lo, hi);
}

// SeedSequence(base + first + i) -> PCG64, one thread per env
__global__ void __launch_bounds__(kThreads) seed_range_kernel(uint64_t *rng, int64_t n, uint32_t b0, uint32_t b1,
                                                              uint32_t b2, uint32_t b3, uint64_t first) {
    const int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    const u128 base = ((u128)b3 << 96) | ((u128)b2 << 64) | ((u128)b1 << 32) | (u128)b0;
    const u128 seed = base + (u128)(first + (uint64_t)i);
    const uint32_t ent[4] = {(uint32_t)seed, (uint32_t)(seed >> 32), (uint32_t)(seed >> 64), (uint32_t)(seed >> 96)};
    Pcg64 g;
    pcg64_from_entropy(g, ent);
    pcg64_store_full(rng + 4 * i, g);
}

__global__ void __launch_bounds__(kThreads) seed_each_kernel(uint64_t *rng, int64_t n, const uint32_t *ent,
                                                             const uint8_t *mask) {
    const int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    if (mask && !mask[i]) return;
    const uint32_t e[4] = {ent[4 * i], ent[4 * i + 1], ent[4 * i + 2], ent[4 * i + 3]};
    Pcg64 g;
    pcg64_from_entropy(g, e);
    pcg64_store_full(rng + 4 * i, g);
}

// [n][S] AoS wire format <-> [S][n] SoA
__global__ void __launch_bounds__(kThreads) state_get_kernel(const double *soa, double *aos, int64_t n, int S) {
    const int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    for (int k = 0; k < S; k++) aos[i * S + k] = soa[k * n + i];
}
__global__ void __launch_bounds__(kThreads) state_set_kernel(double *soa, const double *aos, int64_t n, int S) {
    const int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    for (int k = 0; k < S; k++) soa[k * n + i] = aos[i * S + k];
}

// ---- env snapshots (b200gym_snapshot_*, b200gym_clone) ---------------------------------------------
// One AoS row per env holding every per-env word a later step reads, as 32-bit words:
//   [0, 8)              PCG64 record {state_hi, state_lo, inc_hi, inc_lo}
//   [8, 8 + 2S)         float64 state[S]
//   [8 + 2S, .. + W)    Box2D solver record rec[W] (wind counters and the walker's buffered 32-bit draw included)
//   then elapsed, flags (low byte of a word) and zeros up to a multiple of 32 B (one DRAM sector).
// The transient per-step buffers (toi_mid, the reset / TOI lists) are not state and stay out of the row.
// A CTA moves a tile of T envs through shared memory in 16-byte chunks: thread e takes chunk e / T of env e % T, so
// the lanes of a warp share a chunk (warp-uniform field branches) and read / write each SoA word of 32 consecutive
// envs with one coalesced access.  The tile is contiguous rows of R bytes; R / 16 is even, so a quarter warp's 16-byte
// shared accesses at stride R hit each bank group at most twice (2-way: half the shared bandwidth, still several
// times what HBM can feed).
constexpr int kSnapMaxTileBytes = 96 * 1024;   // opt-in shared memory: 2 CTAs / SM even for the 2 KB hardcore rows

static int snap_record_words(int kind) {
    switch (kind) {
    case B200GYM_LUNARLANDER: case B200GYM_LUNARLANDER_CONT: return lunar::kWords;
    case B200GYM_BIPEDALWALKER: return walker::kWords;
    case B200GYM_BIPEDALWALKER_HARDCORE: return walker::kWordsHC;
    default: return 0;
    }
}
static int snap_unpadded_bytes(int kind) { return 32 + 8 * k_state_dim[kind] + 4 * snap_record_words(kind) + 4 + 1; }
static int snap_row_bytes(int kind) { return (snap_unpadded_bytes(kind) + 31) / 32 * 32; }
static int snap_tile(int row_bytes) {
    int t = kThreads;
    while (t > 32 && t * row_bytes > kSnapMaxTileBytes) t /= 2;
    return t;
}

struct SnapArgs {
    uint32_t *rng, *state, *rec;   // the handle's arrays as 32-bit words
    int32_t *elapsed;
    uint8_t *flags;
    int64_t n;
    int S2, W;                     // 32-bit words of state and of the Box2D record
    int chunks;                    // row bytes / 16
    int tile_log2;                 // T = 1 << tile_log2 envs per CTA
    unsigned long long *bad;       // page-locked, device-mapped word: set by a kernel that meets an out-of-range index
};

__device__ __forceinline__ uint32_t snap_get(const SnapArgs &a, int w, int64_t i) {
    if (w < 8) return a.rng[8 * i + w];
    w -= 8;
    if (w < a.S2) return a.state[2 * ((int64_t)(w >> 1) * a.n + i) + (w & 1)];
    w -= a.S2;
    if (w < a.W) return a.rec[(int64_t)w * a.n + i];
    w -= a.W;
    if (w == 0) return (uint32_t)a.elapsed[i];
    if (w == 1) return a.flags[i];
    return 0u;
}
__device__ __forceinline__ void snap_put(const SnapArgs &a, int w, int64_t i, uint32_t v) {
    if (w < 8) { a.rng[8 * i + w] = v; return; }
    w -= 8;
    if (w < a.S2) { a.state[2 * ((int64_t)(w >> 1) * a.n + i) + (w & 1)] = v; return; }
    w -= a.S2;
    if (w < a.W) { a.rec[(int64_t)w * a.n + i] = v; return; }
    w -= a.W;
    if (w == 0) a.elapsed[i] = (int32_t)v;
    else if (w == 1) a.flags[i] = (uint8_t)v;
}
__device__ __forceinline__ void snap_raise(const SnapArgs &a) {
    *reinterpret_cast<volatile unsigned long long *>(a.bad) = 1ULL;
}

// env idx[k] (idx == NULL: k) -> row k of snap, for k < m.  Out-of-range envs leave a zero row and raise a.bad.
__global__ void __launch_bounds__(kThreads) snapshot_save_kernel(const SnapArgs a, const int64_t *idx, int64_t m,
                                                                 unsigned char *snap) {
    extern __shared__ __align__(128) unsigned char s_tile[];
    const int T = 1 << a.tile_log2, C = a.chunks, R = 16 * C;
    int64_t *s_env = reinterpret_cast<int64_t *>(s_tile + (size_t)T * R);
    const int64_t k0 = (int64_t)blockIdx.x * T;
    const int rows = (int)(m - k0 < T ? m - k0 : T);
    for (int t = threadIdx.x; t < rows; t += kThreads) {
        int64_t i = idx ? idx[k0 + t] : k0 + t;
        if (i < 0 || i >= a.n) { snap_raise(a); i = -1; }
        s_env[t] = i;
    }
    __syncthreads();
    uint4 *tile = reinterpret_cast<uint4 *>(s_tile);
    for (int e = threadIdx.x; e < T * C; e += kThreads) {
        const int t = e & (T - 1), c = e >> a.tile_log2;
        if (t >= rows) continue;
        const int64_t i = s_env[t];
        uint4 v = make_uint4(0u, 0u, 0u, 0u);
        if (i >= 0) {
            v.x = snap_get(a, 4 * c, i); v.y = snap_get(a, 4 * c + 1, i);
            v.z = snap_get(a, 4 * c + 2, i); v.w = snap_get(a, 4 * c + 3, i);
        }
        tile[t * C + c] = v;
    }
    acp::fence_async_smem();
    __syncthreads();
    if (threadIdx.x == 0) {   // the whole tile leaves as one bulk store
        acp::st_bulk(snap + k0 * R, s_tile, (uint32_t)(rows * R));
        acp::st_bulk_commit();
        acp::st_bulk_wait_all();
    }
}

// row row[k] of snap (snap_rows rows) -> env dst[k], for k < m; NULL index arrays = k.  Entries with an out-of-range
// row or env are skipped and raise a.bad.  Duplicate envs in dst: which row lands is undefined.
__global__ void __launch_bounds__(kThreads) snapshot_load_kernel(const SnapArgs a, const unsigned char *snap,
                                                                 int64_t snap_rows, const int64_t *row,
                                                                 const int64_t *dst, int64_t m) {
    extern __shared__ __align__(128) unsigned char s_tile[];
    const int T = 1 << a.tile_log2, C = a.chunks, R = 16 * C;
    int64_t *s_env = reinterpret_cast<int64_t *>(s_tile + (size_t)T * R);
    int64_t *s_row = s_env + T;
    uint64_t *bar = reinterpret_cast<uint64_t *>(s_row + T);
    const int64_t k0 = (int64_t)blockIdx.x * T;
    const int rows = (int)(m - k0 < T ? m - k0 : T);
    for (int t = threadIdx.x; t < rows; t += kThreads) {
        const int64_t r = row ? row[k0 + t] : k0 + t;
        const int64_t d = dst ? dst[k0 + t] : k0 + t;
        const bool ok = r >= 0 && r < snap_rows && d >= 0 && d < a.n;
        if (!ok) snap_raise(a);
        s_row[t] = ok ? r : -1;
        s_env[t] = ok ? d : -1;
    }
    if (threadIdx.x == 0) {
        acp::mbar_init(bar, 1);
        acp::fence_mbar_init();
    }
    __syncthreads();
    if (threadIdx.x < 32) {   // warp 0 gathers the tile's source rows: one bulk copy per row, all completing on `bar`
        const int lane = threadIdx.x;
        int valid = 0;
        for (int t = lane; t < rows; t += 32) valid += s_row[t] >= 0;
        valid = __reduce_add_sync(0xffffffffu, valid);
        if (lane == 0) acp::mbar_arrive_expect_tx(bar, (uint32_t)(valid * R));
        __syncwarp();
        for (int t = lane; t < rows; t += 32)
            if (s_row[t] >= 0) acp::ld_bulk(s_tile + (size_t)t * R, snap + s_row[t] * R, (uint32_t)R, bar);
    }
    acp::mbar_wait(bar, 0);
    const uint4 *tile = reinterpret_cast<const uint4 *>(s_tile);
    for (int e = threadIdx.x; e < T * C; e += kThreads) {
        const int t = e & (T - 1), c = e >> a.tile_log2;
        if (t >= rows) continue;
        const int64_t i = s_env[t];
        if (i < 0) continue;
        const uint4 v = tile[t * C + c];
        snap_put(a, 4 * c, i, v.x); snap_put(a, 4 * c + 1, i, v.y);
        snap_put(a, 4 * c + 2, i, v.z); snap_put(a, 4 * c + 3, i, v.w);
    }
}

// ---- LunarLander-v2 (lunar.cuh): one thread per env, the whole b2World::Step in registers/local ----
constexpr int kLunarThreads = 128;
constexpr int kResetSlots = 64;   // launch ranges of one handle that may be in flight at once (host path: <= 64 chunks)

// lunar_step_kernel runs 128-thread CTAs, but its launch bounds name 256 threads x 2 CTAs: that caps it at 128
// registers, the budget every LunarLander number in DESIGN §4.4 was measured under
constexpr int kLunarRegCapThreads = 256;

// TOI kernels: one warp per CTA, 12 CTAs per SM (what is resident with the 156-register kernel); the kernel strides over
// the list.  Larger grids (fewer envs per warp) are slower (H100 80GB HBM3 at 400 W, 2^16 envs, cold-L2 median):
// LunarLander 1.77 / 1.86 / 1.90 ms at 12 / 64 / 256 CTAs per SM, BipedalWalker (nearly every env parked)
// 8.24 / 11.5 / 16.0 ms
constexpr int kToiCtasPerSm = 12;

// The TOI kernels run one warp per CTA and give each warp as FEW parked envs as the resident grid allows: the lanes
// of a warp diverge completely in this code (different contact lists, GJK / root-finder trip counts, event counts),
// so a warp takes the SUM of its lanes' paths, and with a few thousand parked envs on 132 SMs there are more warp
// slots than envs.  The fewer envs a warp carries, the shorter the launch, down to the floor of ONE env's serial chain
// (up to 5 sub-steps and ~30 b2TimeOfImpact evaluations of dependent, local-memory-heavy code).
__device__ __forceinline__ int toi_lanes_per_warp(int cnt, int nwarps) {
    const int L = (cnt + nwarps - 1) / nwarps;
    return L < 1 ? 1 : (L > 32 ? 32 : L);
}

template <typename ActT, bool CONT>
__global__ void __launch_bounds__(kLunarRegCapThreads, 2) lunar_step_kernel(const StepArgs a) {
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    lunar_step_env<ActT, CONT>(a, j);
}

// The continuous-collision phase of the envs that lunar_step_kernel parked, one warp of parked envs per CTA: the
// TOI code (GJK, root finder, the sub-step solver) is large and runs for a few percent of the envs, so it gets
// its own launch -- dense warps and a warm instruction cache instead of one or two lanes per warp walking it at the
// end of every warp's critical path -- and the warp-synchronous event rounds of b2l::solve_toi.
__global__ void __launch_bounds__(32) lunar_toi_kernel(const StepArgs a) {
    const int cnt = *a.toi_count;
    const int L = toi_lanes_per_warp(cnt, (int)gridDim.x);
    for (int base = blockIdx.x * L; base < cnt; base += gridDim.x * L) {
        const int idx = base + (int)threadIdx.x;
        const bool on = (int)threadIdx.x < L && idx < cnt;
        const unsigned live = __ballot_sync(0xffffffffu, on);
        if (on) lunar_toi_env(a, idx, live);
    }
}

// The autoresets of one step, compacted: a lone finishing env would otherwise keep its whole warp waiting through
// a full reset() (terrain draw + the embedded world step) with one active lane.  Same per-env arithmetic and RNG
// stream as the inline path.
__global__ void __launch_bounds__(kLunarThreads) lunar_reset_list_kernel(const StepArgs a) {
    const int cnt = *a.reset_count;
    for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < cnt; idx += gridDim.x * blockDim.x) lunar_reset_list_env(a, idx);
}

__global__ void __launch_bounds__(kLunarThreads) lunar_reset_kernel(uint32_t *rec, int32_t *elapsed, uint64_t *rng,
                                                                    const uint8_t *mask, float *obs, int64_t n,
                                                                    const lunar::Opts O) {
    const int64_t i = (int64_t)blockIdx.x * kLunarThreads + threadIdx.x;
    if (i >= n) return;
    if (mask && !mask[i]) return;
    float o[8];
    lunar_reset_env(rec, elapsed, rng, n, i, O, o);
    if (obs) store_row<8>(obs, i, o);
}

// wind_idx / torque_idx of every env (lunar_lander.py:234-235): two int32 SoA rows of the record
__global__ void lunar_wind_idx_kernel(uint32_t *rec, int32_t *wind, int32_t *torque, int64_t n, int set) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (set) { rec[(int64_t)lunar::W_WIND * n + i] = (uint32_t)wind[i]; rec[(int64_t)(lunar::W_WIND + 1) * n + i] = (uint32_t)torque[i]; }
    else { wind[i] = (int32_t)rec[(int64_t)lunar::W_WIND * n + i]; torque[i] = (int32_t)rec[(int64_t)(lunar::W_WIND + 1) * n + i]; }
}

// bodies of every env as [n][18] floats {c.x, c.y, a, v.x, v.y, w} x 3 + [n][6] int32 flags (parity harness)
__global__ void lunar_bodies_kernel(const uint32_t *rec, const int32_t *elapsed, float *out, int32_t *flags, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    for (int b = 0; b < 3; b++)
        for (int k = 0; k < 6; k++) out[i * 18 + 6 * b + k] = __uint_as_float(rec[(int64_t)(lunar::W_BODY + 7 * b + k) * n + i]);
    const uint32_t f = rec[(int64_t)lunar::W_FLAGS * n + i];
    int touching = 0;
    for (int sl = 0; sl < lunar::kSlots; sl++) touching += (rec[(int64_t)(lunar::W_SLOT + 7 * sl) * n + i] >> 16) != 0;
    flags[i * 6 + 0] = f & 1u; flags[i * 6 + 1] = (f >> 1) & 1u; flags[i * 6 + 2] = (f >> 2) & 1u;
    flags[i * 6 + 3] = 1; flags[i * 6 + 4] = elapsed[i]; flags[i * 6 + 5] = touching;
}

// envs whose manifold table ever overflowed (b2l::kFlagOverflow in the record's flag word)
__global__ void box2d_overflow_kernel(const uint32_t *flags_row, int64_t n, unsigned long long *count) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && (flags_row[i] & b2l::kFlagOverflow)) atomicAdd(count, 1ULL);
}

static int lunar_upload_consts(b200gym *h) {
    lunar::Consts c;
    b2l_host::lunar_consts(c);
    CK(h, cudaMemcpyToSymbol(lunar::kC, &c, sizeof c));
    return 0;
}

// ---- BipedalWalker-v3 (walker.cuh): one thread per env --------------------------------------------
template <bool HC>
__global__ void __launch_bounds__(kLunarThreads, 4) walker_step_kernel(const StepArgs a) {
    const int64_t j = (int64_t)blockIdx.x * kLunarThreads + threadIdx.x;
    if (j < a.count) walker_step_env<HC>(a, j);
}

// the continuous-collision phase of the parked envs (see lunar_toi_kernel)
template <bool HC>
__global__ void __launch_bounds__(32) walker_toi_kernel(const StepArgs a) {
    const int cnt = *a.toi_count;
    const int L = toi_lanes_per_warp(cnt, (int)gridDim.x);
    for (int base = blockIdx.x * L; base < cnt; base += gridDim.x * L) {
        const int idx = base + (int)threadIdx.x;
        const bool on = (int)threadIdx.x < L && idx < cnt;
        const unsigned live = __ballot_sync(0xffffffffu, on);
        if (on) walker_toi_env<HC>(a, idx, live);
    }
}

template <bool HC>
__global__ void __launch_bounds__(kLunarThreads, 4) walker_reset_list_kernel(const StepArgs a) {
    const int cnt = *a.reset_count;
    for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < cnt; idx += gridDim.x * blockDim.x) walker_reset_list_env<HC>(a, idx);
}

template <bool HC>
__global__ void __launch_bounds__(kLunarThreads) walker_reset_kernel(uint32_t *rec, int32_t *elapsed, uint64_t *rng,
                                                                     const uint8_t *mask, float *obs, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * kLunarThreads + threadIdx.x;
    if (i >= n) return;
    if (mask && !mask[i]) return;
    float o[24];
    walker_reset_env<HC>(rec, elapsed, rng, n, i, o);
    if (obs) store_row<24>(obs, i, o);
}

// a fresh Generator has an empty 32-bit cache: clear {has_uint32, uinteger} of the (re)seeded envs
__global__ void walker_clear_rng32_kernel(uint32_t *rec, const uint8_t *mask, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || (mask && !mask[i])) return;
    rec[(int64_t)walker::W_RNG32 * n + i] = 0u;
    rec[(int64_t)(walker::W_RNG32 + 1) * n + i] = 0u;
}

// terrain heights [n][200] and (hardcore) obstacle boxes [n][40][4] = {x0, ylo, x1, yhi} + their number [n]
__global__ void walker_terrain_kernel(const uint32_t *rec, float *terrain, float *polys, int32_t *npoly, int64_t n, int hardcore) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    for (int k = 0; k < walker::kTerrain; k++) terrain[i * walker::kTerrain + k] = __uint_as_float(rec[(int64_t)(walker::W_TERRAIN + k) * n + i]);
    if (!polys || !npoly) return;
    const int np = hardcore ? (int)rec[(int64_t)walker::W_NPOLY * n + i] : 0;
    npoly[i] = np;
    for (int k = 0; k < 4 * walker::NP; k++)
        polys[i * 4 * walker::NP + k] = k < 4 * np ? __uint_as_float(rec[(int64_t)(walker::W_POLY + k) * n + i]) : 0.0f;
}

__global__ void walker_bodies_kernel(const uint32_t *rec, float *out, int32_t *flags, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    for (int b = 0; b < walker::NB; b++)
        for (int k = 0; k < 6; k++) out[i * 30 + 6 * b + k] = __uint_as_float(rec[(int64_t)(walker::W_BODY + 7 * b + k) * n + i]);
    const uint32_t f = rec[(int64_t)walker::W_FLAGS * n + i];
    int touching = 0;
    for (int sl = 0; sl < walker::kSlots; sl++) touching += (rec[(int64_t)(walker::W_SLOT + 7 * sl) * n + i] >> 16) != 0;
    flags[i * 4 + 0] = f & 1u; flags[i * 4 + 1] = (f >> 1) & 1u; flags[i * 4 + 2] = (f >> 2) & 1u; flags[i * 4 + 3] = touching;
}

static int walker_upload_consts(b200gym *h) {
    walker::Consts c;
    b2l_host::walker_consts(c);
    CK(h, cudaMemcpyToSymbol(walker::kC, &c, sizeof c));
    return 0;
}

// ---- SURVEY.md 8(f): vector-aware wrappers fused on the device ---------------------------------------
// RecordEpisodeStatistics (gym/wrappers/record_episode_statistics.py:103-151): the reference walks the
// batch in a Python loop; here one launch updates the float32 return / int32 length accumulators,
// emits infos["episode"]["r"/"l"] + the `_episode` mask, and appends finished episodes to a small ring
// (the return_queue / length_queue deques).
__global__ void __launch_bounds__(kThreads) episode_stats_kernel(const double *reward, const uint8_t *term,
                                                                const uint8_t *trunc, float *ret_acc, int32_t *len_acc,
                                                                float *ep_r, int32_t *ep_l, uint8_t *ep_mask,
                                                                unsigned long long *ring,
                                                                unsigned long long *counter, int ring_size, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    // `self.episode_returns += rewards` on a float32 array with float64 rewards: add in float64, round to float32
    const float ret = (float)((double)ret_acc[i] + reward[i]);
    const int32_t len = len_acc[i] + 1;
    const bool done = term[i] | trunc[i];
    ep_mask[i] = done ? 1 : 0;
    if (done) {
        ep_r[i] = ret;
        ep_l[i] = len;
        if (ring_size > 0) {
            // one 64-bit store per episode {length : return bits}: when more than ring_size episodes finish in one
            // step several of them land on the same slot, and a slot must never mix two episodes
            const unsigned long long slot = atomicAdd(counter, 1ULL);
            ring[slot % (unsigned long long)ring_size] =
                ((unsigned long long)(uint32_t)len << 32) | (unsigned long long)__float_as_uint(ret);
        } else atomicAdd(counter, 1ULL);
        ret_acc[i] = 0.0f;
        len_acc[i] = 0;
    } else {
        ret_acc[i] = ret;
        len_acc[i] = len;
    }
}

// NormalizeObservation / NormalizeReward (gym/wrappers/normalize.py:8-144): RunningMeanStd over the batch axis,
// two launches per step and ONE pass over the batch for the moments.
//   launch 1 (moments): the batch is read as a flat [n*D] stream; the CTA size is a multiple of D, so every
//     thread stays on one column and the loads are perfectly coalesced whatever D is.  Per column: sum and sum of
//     squares of the deviations from a pivot (the current running mean: numerically tame), float64.  The sums are
//     reduced in a fixed order, so a launch is reproducible bit for bit: a tree over the CTA's threads of each
//     column, one partial per CTA and column in the workspace, and the last CTA to take the ticket adds the
//     partials in CTA order (strided over its threads, then the same tree) into scratch.  The order depends on n
//     and D only.
//   (between the launches a sharded env all-reduces the 2*D sums across GPUs: torch.distributed, 8 * 2 * D bytes)
//   launch 2 (apply): every CTA folds the batch moments into the running ones (Chan et al., normalize.py:32-46) on
//     its own -- D <= 24 columns, a few dozen flops -- normalises its share of the batch with the NEW statistics
//     (normalize.py:83-95) and CTA 0 publishes them.  Statistics and scratch are double-buffered by step parity, so
//     no CTA can read a half-updated value.
// stats layout (float64, caller-owned): [2][2*D + 1] = {mean[D], var[D], count}; scratch: [2][2*D] = {sum[D], sumsq[D]};
// work: [1 + 2*D*kNormMaxCtas] = {CTA ticket (zero bits between launches), partials[CTA][2*D]}.
constexpr int kMaxNormDim = 24;
constexpr int kNormMaxCtas = B200GYM_RMS_MAX_CTAS;
constexpr int kNormMaxBlock = 256;

// sh[.][c + D*j], j < blockDim.x / D (a power of two for every accepted D) -> sh[.][c], pairs at a fixed distance
__device__ __forceinline__ void norm_tree(double (*sh)[kNormMaxBlock], int D) {
    const int tid = threadIdx.x;
    for (int h = blockDim.x / D / 2; h > 0; h >>= 1) {
        if (tid < h * D) {
            sh[0][tid] += sh[0][tid + h * D];
            sh[1][tid] += sh[1][tid + h * D];
        }
        __syncthreads();
    }
}

template <typename T, bool RETURNS>
__global__ void __launch_bounds__(kNormMaxBlock) rms_moments_kernel(const T *x, double *returns, const double *reward,
                                                                    double gamma, int64_t total, int D,
                                                                    const double *stats, double *scratch, double *work) {
    __shared__ double sh[2][kNormMaxBlock];
    __shared__ bool last;
    const int tid = threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;      // a multiple of D: the column of a thread is fixed
    const int64_t start = (int64_t)blockIdx.x * blockDim.x + tid;
    const int col = tid % D;                                     // = start % D: blockDim.x is a multiple of D
    const double pivot = stats[col];
    double s = 0.0, q = 0.0;
    for (int64_t k = start; k < total; k += stride) {
        double v;
        if constexpr (RETURNS) {   // NormalizeReward.step (normalize.py:130): returns = returns * gamma + reward
            v = returns[k] * gamma + reward[k];
            returns[k] = v;
        } else {
            v = (double)x[k];
        }
        v -= pivot;
        s += v;
        q += v * v;
    }
    sh[0][tid] = s;
    sh[1][tid] = q;
    __syncthreads();
    norm_tree(sh, D);
    unsigned int *ticket = reinterpret_cast<unsigned int *>(work);
    double *partials = work + 1;
    if (tid < D) {
        partials[(int64_t)blockIdx.x * 2 * D + tid] = sh[0][tid];
        partials[(int64_t)blockIdx.x * 2 * D + D + tid] = sh[1][tid];
        __threadfence();                                         // the partials are visible before the ticket is taken
    }
    __syncthreads();
    if (tid == 0) last = atomicAdd(ticket, 1u) == gridDim.x - 1;
    __syncthreads();
    if (!last) return;
    __threadfence();
    // the last CTA: thread tid adds the partials of CTAs tid / D, tid / D + m, ... in order (m = blockDim.x / D)
    s = 0.0;
    q = 0.0;
    for (int b = tid / D; b < (int)gridDim.x; b += blockDim.x / D) {
        s += __ldcg(&partials[(int64_t)b * 2 * D + col]);
        q += __ldcg(&partials[(int64_t)b * 2 * D + D + col]);
    }
    sh[0][tid] = s;
    sh[1][tid] = q;
    __syncthreads();
    norm_tree(sh, D);
    if (tid < D) {
        scratch[tid] += sh[0][tid];
        scratch[D + tid] += sh[1][tid];
    }
    if (tid == 0) *ticket = 0u;                                  // ready for the next launch (stream order)
}

// update_mean_var_count_from_moments (normalize.py:32-46) for column d, from the pivoted batch sums
__device__ __forceinline__ void chan_update(const double *stats, const double *scratch, int D, int d, double bn, double &mean,
                                            double &var, double &count) {
    const double dm = scratch[d] / bn;                 // batch_mean - pivot (pivot = old mean) = delta
    const double batch_var = scratch[D + d] / bn - dm * dm;
    const double cnt = stats[2 * D];
    const double tot = cnt + bn;
    mean = stats[d] + dm * bn / tot;
    const double m2 = stats[D + d] * cnt + batch_var * bn + dm * dm * cnt * bn / tot;
    var = m2 / tot;
    count = tot;
}

template <bool REWARD>
__global__ void rms_apply_kernel(const float *x, float *out, const double *reward, double *out_r, double *returns,
                                 const uint8_t *term, const uint8_t *trunc, int64_t total, int D, const double *stats,
                                 double *stats_next, const double *scratch, double *scratch_next, double batch_count,
                                 double eps, int update) {
    __shared__ double sh_mean[kMaxNormDim], sh_inv[kMaxNormDim];
    const int tid = threadIdx.x;
    if (tid < D) {
        double mean = stats[tid], var = stats[D + tid], count = stats[2 * D];
        if (update) chan_update(stats, scratch, D, tid, batch_count, mean, var, count);
        sh_mean[tid] = mean;
        sh_inv[tid] = sqrt(var + eps);
        if (blockIdx.x == 0 && update) {
            stats_next[tid] = mean;
            stats_next[D + tid] = var;
            if (tid == 0) stats_next[2 * D] = count;
            scratch_next[tid] = 0.0;                   // next step accumulates into the other scratch buffer
            scratch_next[D + tid] = 0.0;
        }
    }
    __syncthreads();
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    const int64_t start = (int64_t)blockIdx.x * blockDim.x + tid;
    const int col = (int)(start % D);
    const double mean = sh_mean[col], sd = sh_inv[col];
    for (int64_t k = start; k < total; k += stride) {
        if constexpr (REWARD) {
            out_r[k] = reward[k] / sd;                                 // normalize.py:143 (no mean subtraction)
            if (term[k] | trunc[k]) returns[k] = 0.0;                  // :135-136
        } else {
            out[k] = (float)(((double)x[k] - mean) / sd);              // normalize.py:95
        }
    }
}

// The normalised rows x[n][D] of observation rows o[n][D] (norm_obs_elem), one thread per element: the input rows of
// the Box2D kinds' policy and critic launches when the observations are normalised
__global__ void __launch_bounds__(kThreads) norm_rows_kernel(const float *o, float *x, int64_t total, int D,
                                                             const ObsNormArgs q) {
    __shared__ double mean[kMaxNormDim], sd[kMaxNormDim];
    if (threadIdx.x < D) {
        mean[threadIdx.x] = q.mean[threadIdx.x];
        sd[threadIdx.x] = norm_sd(q.var[threadIdx.x], q.eps);
    }
    __syncthreads();
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k < total) x[k] = norm_obs_elem(o[k], mean[k % D], sd[k % D], q.clip);
}

// ---- cross-GPU step barrier for the fused all-gather ---------------------------------------
// flags[r] (uint64, in every rank's gather allocation) = number of steps whose results rank r has fully written
// into THIS rank's buffers.  One launch per step, after the step kernel on the same stream: lane p publishes
// "my rows of step k are in your buffers" to peer p (the kernel boundary has drained the step kernel's stores,
// bulk ones included; the system-scope fence orders them before the flag) and then waits for peer p's flag.
// A peer that died does not hang the stream for ever: after `timeout_ns` the lane records the peer in
// `*timed_out` (sticky, read by b200gym_p2p_status) and gives up.
__global__ void p2p_sync_kernel(unsigned long long *const *peer_flags, const unsigned long long *my_flags, int world,
                                int rank, unsigned long long step, unsigned long long timeout_ns, int *timed_out) {
    const int p = threadIdx.x;
    if (p < world && p != rank) {
        __threadfence_system();
        volatile unsigned long long *f = peer_flags[p] + rank;
        *f = step;
        const volatile unsigned long long *w = my_flags + p;
        const unsigned long long t0 = global_ns();
        while (*w < step) {
            if (global_ns() - t0 > timeout_ns) {
                atomicExch(timed_out, p + 1);
                break;
            }
        }
        __threadfence_system();
    }
}

// device self-test: div_by_const(x, c, RN(1/c)) must equal x / c bit for bit
__global__ void __launch_bounds__(kThreads) selftest_div_kernel(int64_t samples, uint64_t seed,
                                                                unsigned long long *mismatches) {
    const double cs[4] = {1.1, 0.1 + 1.0, 3.0, 9.8};
    const int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= samples) return;
    // splitmix64 bits -> doubles spread over many binades, both signs
    uint64_t z = seed + 0x9E3779B97F4A7C15ULL * (uint64_t)(i + 1);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
    z ^= z >> 31;
    const double mant = 1.0 + (double)(z >> 12) * (1.0 / 4503599627370496.0);
    const int e = (int)((z >> 3) & 0x3F) - 32;
    double x = ldexp(mant, e);
    if (z & 1) x = -x;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const double c = cs[k];
        const double rc = 1.0 / c;
        const double fast = div_by_const(x, c, rc);
        const double ref = x / c;
        if (__double_as_longlong(fast) != __double_as_longlong(ref)) atomicAdd(mismatches, 1ULL);
    }
}

// device self-test: csrc/glibc_trig.cuh evaluated on caller-supplied arguments (the host compares with its libm)
__global__ void __launch_bounds__(kThreads) selftest_trig_kernel(const double *x, int64_t n, double *sn, double *cs, double *sq) {
    const int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    sn[i] = gt::sin(x[i]);
    cs[i] = gt::cos(x[i]);
    if (sq) sq[i] = gt::sq(x[i]);
}

// device self-test: the tanh activation of the MLP policies (mlp_tanh) evaluated on caller-supplied arguments (the
// caller compares with torch.tanh on the same device)
__global__ void __launch_bounds__(kThreads) selftest_tanh_kernel(const float *x, int64_t n, float *y) {
    const int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    y[i] = mlp_tanh(x[i]);
}

// device self-test: the exp of the SAC head (head_exp) evaluated on caller-supplied arguments (the caller compares
// with torch.exp on the same device)
__global__ void __launch_bounds__(kThreads) selftest_exp_kernel(const float *x, int64_t n, float *y) {
    const int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    y[i] = head_exp(x[i]);
}

static inline unsigned blocks_for(int64_t n) { return (unsigned)((n + kThreads - 1) / kThreads); }

// ---------------------------------------------------------------------------
// dispatch
// ---------------------------------------------------------------------------
// Kernel B by default where it measured faster than kernel P (DESIGN §4.1): CartPole, at 2^18, 2^20 and 2^23 envs.  The other
// kinds are slower with it at 2^18 envs -- one partly filled wave, latency-bound, where B's 32 compute warps per SM
// (P: 48) cost more than moving the memory traffic off the compute warps saves
static bool bulk_by_default(int kind) { return kind == B200GYM_CARTPOLE; }

template <typename ActT>
static constexpr int act_width_slot() { return sizeof(ActT) == 8 ? 0 : sizeof(ActT) == 4 ? 1 : 2; }

// The resident kernels' CTAs per SM (and kernel B's shared-memory attributes) for one action type, set up when the
// handle is created rather than on its first step: that step may be the one a CUDA graph captures, and the capture
// must hold nothing but launches
template <int KIND, typename ActT>
static int prepare_step_typed(b200gym *h) {
    const int w = act_width_slot<ActT>();
    if (h->kernel_choice == 2 || (h->kernel_choice == -1 && bulk_by_default(KIND))) {
        const int smem = kBulkStages * BulkLayout<KIND, ActT>::kBytes;
        int &occ = h->occ_bulk[KIND][w];
        CK(h, cudaFuncSetAttribute(step_kernel_persistent_bulk<KIND, ActT>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        CK(h, cudaFuncSetAttribute(step_kernel_persistent_bulk<KIND, ActT>, cudaFuncAttributePreferredSharedMemoryCarveout,
                                   (int)cudaSharedmemCarveoutMaxShared));
        CK(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, step_kernel_persistent_bulk<KIND, ActT>, kThreads + 32, smem));
        if (occ < 1) occ = 1;
    }
    if (h->kernel_choice != 0) {
        int &occ = h->occ[KIND][w];
        CK(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, step_kernel_persistent<KIND, ActT>, kThreads, 0));
        if (occ < 1) occ = 1;
    }
    return 0;
}

template <int KIND>
static int prepare_step_kind(b200gym *h) {
    if constexpr (Env<KIND>::A == 0)
        return prepare_step_typed<KIND, long long>(h) || prepare_step_typed<KIND, int>(h) ||
               prepare_step_typed<KIND, unsigned char>(h);
    else
        return prepare_step_typed<KIND, float>(h);
}

static int prepare_step(b200gym *h) {
    switch (h->cfg.kind) {
    case B200GYM_CARTPOLE: return prepare_step_kind<B200GYM_CARTPOLE>(h);
    case B200GYM_MOUNTAINCAR: return prepare_step_kind<B200GYM_MOUNTAINCAR>(h);
    case B200GYM_MOUNTAINCAR_CONT: return prepare_step_kind<B200GYM_MOUNTAINCAR_CONT>(h);
    case B200GYM_PENDULUM: return prepare_step_kind<B200GYM_PENDULUM>(h);
    case B200GYM_ACROBOT: return prepare_step_kind<B200GYM_ACROBOT>(h);
    }
    return 0;   // the Box2D tasks' kernels need no set-up
}

template <int KIND, typename ActT>
static int launch_step_typed(b200gym *h, const StepArgs &a, cudaStream_t st) {
    int64_t done = 0;
    const int64_t tiles = a.count / kThreads;
    if ((a.npeer > 0 || a.bulk_sink) && tiles > 0) {
        // kernel G (bulk pushes): every destination row block must be 16-byte aligned
        auto ok = [&](const float *o, const double *r, const uint8_t *te, const uint8_t *tr) {
            return (uintptr_t)(o + a.first * Env<KIND>::D) % 16 == 0 && (uintptr_t)(r + a.first) % 16 == 0 &&
                   (uintptr_t)(te + a.first) % 16 == 0 && (uintptr_t)(tr + a.first) % 16 == 0;
        };
        bool aligned = ok(a.obs, a.reward, a.terminated, a.truncated);
        for (int p = 0; p < a.npeer; p++) aligned = aligned && ok(a.peer_obs[p], a.peer_reward[p], a.peer_term[p], a.peer_trunc[p]);
        if (aligned) {
            StepArgs g = a;
            // the fused step barrier needs the whole range in this one launch (a ragged tail goes through kernel A,
            // whose stores the barrier would not cover): otherwise b200gym_step_p2p launches p2p_sync_kernel
            const bool fused_barrier = a.p2p_done != nullptr && tiles * kThreads == a.count;
            if (!fused_barrier) g.p2p_done = nullptr;
            step_kernel_gather<KIND, ActT><<<(unsigned)tiles, kThreads, 0, st>>>(g);
            CK(h, cudaGetLastError());
            done = tiles * kThreads;
            h->p2p_barrier_fused = fused_barrier;
        }
    }
    // the resident kernels index envs in 32 bits; larger handles step on kernel A
    const bool resident = a.npeer == 0 && a.count >= (int64_t)h->sm_count * kThreads && h->n < (int64_t)1 << 30;
    const bool bulk = h->kernel_choice == 2 || (h->kernel_choice == -1 && bulk_by_default(KIND));
    if (done == 0 && resident && bulk) {
        // kernel B: whole tiles, every row a bulk copy touches 16-byte aligned
        using L = BulkLayout<KIND, ActT>;
        const auto al = [](const void *p) { return (uintptr_t)p % 16 == 0; };
        bool aligned = h->n % 2 == 0 && al(a.state + a.first) && al(a.elapsed + a.first) && al(a.obs + a.first * Env<KIND>::D) &&
                       al(a.reward + a.first) && al(a.terminated + a.first) && al(a.truncated + a.first) &&
                       al(reinterpret_cast<const ActT *>(a.actions) + a.first * L::kActPerEnv);
        if (aligned) {
            const int smem = kBulkStages * L::kBytes;
            const int occ = h->occ_bulk[KIND][act_width_slot<ActT>()];   // prepare_step_typed, at create
            int64_t grid = (int64_t)h->sm_count * occ;
            if (grid > tiles) grid = tiles;
            step_kernel_persistent_bulk<KIND, ActT><<<(unsigned)grid, kThreads + 32, smem, st>>>(a, (int)tiles);
            CK(h, cudaGetLastError());
            done = tiles * kThreads;   // a ragged tail goes to kernel A below
        }
    }
    if (done == 0 && h->kernel_choice != 0 && resident) {
        // kernel P: resident grid; needs naturally aligned input words for cp.async (always true for the
        // handle's own arrays; the caller's action pointer is checked)
        using L = PrefetchLayout<KIND, ActT>;
        const bool aligned = !L::kActAsync || ((uintptr_t)a.actions % L::kActBytes == 0);
        if (aligned) {
            const int occ = h->occ[KIND][act_width_slot<ActT>()];   // prepare_step_typed, at create
            const int64_t all_tiles = (a.count + kThreads - 1) / kThreads;
            int64_t grid = (int64_t)h->sm_count * occ;
            if (grid > all_tiles) grid = all_tiles;
            step_kernel_persistent<KIND, ActT><<<(unsigned)grid, kThreads, 0, st>>>(a, (int)all_tiles);
            CK(h, cudaGetLastError());
            done = a.count;
        }
    }
    if (done < a.count) {
        StepArgs t = a;
        t.first = a.first + done;
        t.count = a.count - done;
        step_kernel<KIND, ActT><<<blocks_for(t.count), kThreads, 0, st>>>(t);
        CK(h, cudaGetLastError());
    }
    return 0;
}

template <int KIND>
static int launch_step_kind(b200gym *h, const StepArgs &a, int action_dtype, cudaStream_t st) {
    using E = Env<KIND>;
    if constexpr (E::A == 0) {
        switch (action_dtype) {
        case B200GYM_ACT_I64: return launch_step_typed<KIND, long long>(h, a, st);
        case B200GYM_ACT_I32: return launch_step_typed<KIND, int>(h, a, st);
        case B200GYM_ACT_U8: return launch_step_typed<KIND, unsigned char>(h, a, st);
        default: return fail(h, "Discrete env needs an integer action dtype (got code %d)", action_dtype);
        }
    } else {
        if (action_dtype != B200GYM_ACT_F32)
            return fail(h, "Box env needs float32 actions (got dtype code %d)", action_dtype);
        return launch_step_typed<KIND, float>(h, a, st);
    }
}

// A Box2D step: step kernel -> TOI kernel over the parked envs -> compacted reset-list kernel; the last two only when
// their path is deferred (else the step kernel solves TOI / resets inline)
static int launch_step_box2d(b200gym *h, const StepArgs &a, int action_dtype, cudaStream_t st) {
    using Kernel = void (*)(const StepArgs);
    Kernel step, toi, reset_list;
    if (h->is_lunar) {
        if (h->cfg.kind == B200GYM_LUNARLANDER_CONT) {
            if (action_dtype != B200GYM_ACT_F32) return fail(h, "Box env needs float32 actions (got dtype code %d)", action_dtype);
            if ((uintptr_t)a.actions % 8 != 0) return fail(h, "LunarLanderContinuous actions must be 8-byte aligned");
            step = lunar_step_kernel<float, true>;
        } else {
            switch (action_dtype) {
            case B200GYM_ACT_I64: step = lunar_step_kernel<long long, false>; break;
            case B200GYM_ACT_I32: step = lunar_step_kernel<int, false>; break;
            case B200GYM_ACT_U8: step = lunar_step_kernel<unsigned char, false>; break;
            default: return fail(h, "Discrete env needs an integer action dtype (got code %d)", action_dtype);
            }
        }
        toi = lunar_toi_kernel;
        reset_list = lunar_reset_list_kernel;
    } else {
        if (action_dtype != B200GYM_ACT_F32) return fail(h, "Box env needs float32 actions (got dtype code %d)", action_dtype);
        if ((uintptr_t)a.actions % 16 != 0) return fail(h, "BipedalWalker actions must be 16-byte aligned");
        const bool hc = h->cfg.kind == B200GYM_BIPEDALWALKER_HARDCORE;
        step = hc ? walker_step_kernel<true> : walker_step_kernel<false>;
        toi = hc ? walker_toi_kernel<true> : walker_toi_kernel<false>;
        reset_list = hc ? walker_reset_list_kernel<true> : walker_reset_list_kernel<false>;
    }
    StepArgs b = a;
    const bool defer = h->cfg.autoreset && h->box2d_defer && h->reset_list;
    if (defer) {   // the caller may have picked a counter slot (one per concurrently running range)
        b.reset_list = h->reset_list;
        if (!b.reset_count) b.reset_count = h->reset_count;
        CK(h, cudaMemsetAsync(b.reset_count, 0, sizeof(int32_t), st));
    } else {
        b.reset_list = nullptr; b.reset_count = nullptr;
    }
    // continuous collision of the parked envs in its own launch (see lunar_toi_kernel)
    const bool toi_defer = h->box2d_toi_defer && h->toi_list;
    if (toi_defer) {
        b.toi_list = h->toi_list;
        b.toi_mid = h->toi_mid;
        if (!b.toi_count) b.toi_count = h->toi_count;
        CK(h, cudaMemsetAsync(b.toi_count, 0, sizeof(int32_t), st));
    } else {
        b.toi_list = nullptr; b.toi_count = nullptr; b.toi_mid = nullptr;
    }
    const int64_t blocks = (b.count + kLunarThreads - 1) / kLunarThreads;
    step<<<(unsigned)blocks, kLunarThreads, 0, st>>>(b);
    CK(h, cudaGetLastError());
    if (toi_defer) {
        toi<<<(unsigned)std::min<int64_t>(b.count, (int64_t)kToiCtasPerSm * h->sm_count), 32, 0, st>>>(b);
        CK(h, cudaGetLastError());
    }
    // at most 2 CTAs per SM of the compacted reset kernel (it strides over the list)
    if (defer) reset_list<<<(unsigned)std::min<int64_t>(blocks, 2 * h->sm_count), kLunarThreads, 0, st>>>(b);
    CK(h, cudaGetLastError());
    return 0;
}

static int launch_step(b200gym *h, const StepArgs &a, int action_dtype, cudaStream_t st) {
    switch (h->cfg.kind) {
    case B200GYM_CARTPOLE: return launch_step_kind<B200GYM_CARTPOLE>(h, a, action_dtype, st);
    case B200GYM_MOUNTAINCAR: return launch_step_kind<B200GYM_MOUNTAINCAR>(h, a, action_dtype, st);
    case B200GYM_MOUNTAINCAR_CONT: return launch_step_kind<B200GYM_MOUNTAINCAR_CONT>(h, a, action_dtype, st);
    case B200GYM_PENDULUM: return launch_step_kind<B200GYM_PENDULUM>(h, a, action_dtype, st);
    case B200GYM_ACROBOT: return launch_step_kind<B200GYM_ACROBOT>(h, a, action_dtype, st);
    case B200GYM_LUNARLANDER:
    case B200GYM_LUNARLANDER_CONT:
    case B200GYM_BIPEDALWALKER:
    case B200GYM_BIPEDALWALKER_HARDCORE: return launch_step_box2d(h, a, action_dtype, st);
    }
    return fail(h, "bad kind %d", h->cfg.kind);
}

template <int KIND>
static int launch_rollout_kind(b200gym *h, const StepArgs &a, int action_dtype, int32_t T, float *last_obs,
                               cudaStream_t st) {
    if constexpr (Env<KIND>::A == 0) {
        switch (action_dtype) {
        case B200GYM_ACT_I64: rollout_kernel<KIND, long long><<<blocks_for(h->n), kThreads, 0, st>>>(a, T, last_obs); break;
        case B200GYM_ACT_I32: rollout_kernel<KIND, int><<<blocks_for(h->n), kThreads, 0, st>>>(a, T, last_obs); break;
        case B200GYM_ACT_U8: rollout_kernel<KIND, unsigned char><<<blocks_for(h->n), kThreads, 0, st>>>(a, T, last_obs); break;
        default: return fail(h, "Discrete env needs an integer action dtype (got code %d)", action_dtype);
        }
    } else {
        if (action_dtype != B200GYM_ACT_F32) return fail(h, "Box env needs float32 actions (got dtype code %d)", action_dtype);
        rollout_kernel<KIND, float><<<blocks_for(h->n), kThreads, 0, st>>>(a, T, last_obs);
    }
    CK(h, cudaGetLastError());
    return 0;
}

static size_t action_size(int action_dtype);

// A Box2D rollout: the step sequence of launch_step_box2d once per step, into slice t; those steps are bound by
// their arithmetic (milliseconds at 2^16 envs), so keeping the state on chip would save nothing measurable
static int launch_rollout_box2d(b200gym *h, const StepArgs &a, int action_dtype, int32_t T, float *last_obs,
                                cudaStream_t st) {
    const int64_t n = h->n, D = h->D;
    const size_t act_row = (size_t)n * std::max(h->A, 1) * action_size(action_dtype);
    StepArgs s = a;
    for (int32_t t = 0; t < T; t++) {
        s.actions = static_cast<const unsigned char *>(a.actions) + (size_t)t * act_row;
        s.obs = a.obs + t * n * D;
        s.reward = a.reward + t * n;
        s.terminated = a.terminated + t * n;
        s.truncated = a.truncated + t * n;
        s.final_obs = a.final_obs ? a.final_obs + t * n * D : nullptr;
        if (launch_step_box2d(h, s, action_dtype, st)) return 1;
    }
    CK(h, cudaMemcpyAsync(last_obs, s.obs, (size_t)n * D * sizeof(float), cudaMemcpyDeviceToDevice, st));
    return 0;
}

static int launch_rollout(b200gym *h, const StepArgs &a, int action_dtype, int32_t T, float *last_obs, cudaStream_t st) {
    switch (h->cfg.kind) {
    case B200GYM_CARTPOLE: return launch_rollout_kind<B200GYM_CARTPOLE>(h, a, action_dtype, T, last_obs, st);
    case B200GYM_MOUNTAINCAR: return launch_rollout_kind<B200GYM_MOUNTAINCAR>(h, a, action_dtype, T, last_obs, st);
    case B200GYM_MOUNTAINCAR_CONT: return launch_rollout_kind<B200GYM_MOUNTAINCAR_CONT>(h, a, action_dtype, T, last_obs, st);
    case B200GYM_PENDULUM: return launch_rollout_kind<B200GYM_PENDULUM>(h, a, action_dtype, T, last_obs, st);
    case B200GYM_ACROBOT: return launch_rollout_kind<B200GYM_ACROBOT>(h, a, action_dtype, T, last_obs, st);
    case B200GYM_LUNARLANDER:
    case B200GYM_LUNARLANDER_CONT:
    case B200GYM_BIPEDALWALKER:
    case B200GYM_BIPEDALWALKER_HARDCORE: return launch_rollout_box2d(h, a, action_dtype, T, last_obs, st);
    }
    return fail(h, "bad kind %d", h->cfg.kind);
}

template <int KIND>
static void launch_reset_kind(b200gym *h, const uint8_t *mask, const double *bounds, float *obs, cudaStream_t st) {
    double lo, hi;
    Env<KIND>::default_bounds(lo, hi);
    if (bounds) { lo = bounds[0]; hi = bounds[1]; }
    reset_kernel<KIND><<<blocks_for(h->n), kThreads, 0, st>>>(h->state, h->elapsed, h->flags, h->rng, mask, obs,
                                                              h->n, lo, hi);
}

static int launch_reset(b200gym *h, const uint8_t *mask, const double *bounds, float *obs, cudaStream_t st) {
    switch (h->cfg.kind) {
    case B200GYM_CARTPOLE: launch_reset_kind<B200GYM_CARTPOLE>(h, mask, bounds, obs, st); break;
    case B200GYM_MOUNTAINCAR: launch_reset_kind<B200GYM_MOUNTAINCAR>(h, mask, bounds, obs, st); break;
    case B200GYM_MOUNTAINCAR_CONT: launch_reset_kind<B200GYM_MOUNTAINCAR_CONT>(h, mask, bounds, obs, st); break;
    case B200GYM_PENDULUM: launch_reset_kind<B200GYM_PENDULUM>(h, mask, bounds, obs, st); break;
    case B200GYM_ACROBOT: launch_reset_kind<B200GYM_ACROBOT>(h, mask, bounds, obs, st); break;
    case B200GYM_LUNARLANDER:
    case B200GYM_LUNARLANDER_CONT:
        lunar_reset_kernel<<<(unsigned)((h->n + kLunarThreads - 1) / kLunarThreads), kLunarThreads, 0, st>>>(
            h->lunar_rec, h->elapsed, h->rng, mask, obs, h->n, h->lunar_opts);
        break;
    case B200GYM_BIPEDALWALKER:
        walker_reset_kernel<false><<<(unsigned)((h->n + kLunarThreads - 1) / kLunarThreads), kLunarThreads, 0, st>>>(
            h->lunar_rec, h->elapsed, h->rng, mask, obs, h->n);
        break;
    case B200GYM_BIPEDALWALKER_HARDCORE:
        walker_reset_kernel<true><<<(unsigned)((h->n + kLunarThreads - 1) / kLunarThreads), kLunarThreads, 0, st>>>(
            h->lunar_rec, h->elapsed, h->rng, mask, obs, h->n);
        break;
    default: return fail(h, "bad kind %d", h->cfg.kind);
    }
    CK(h, cudaGetLastError());
    return 0;
}

// ---------------------------------------------------------------------------
// space_sample_kernel: `envs.action_space.sample()` of the batched action space (space_sample.cuh: one 16-byte
// vector per thread and round, grid-strided; a table jump to the first vector, one multiply-add to each next one)
// ---------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kSampleThreads) space_sample_kernel(const SampleArgs a, T *__restrict__ out) {
    __shared__ LcgJumpTable table;   // rows [0, jump_digits) of kLcgJump, 512 B each
    const uint4 *src = reinterpret_cast<const uint4 *>(&kLcgJump);
    uint4 *dst = reinterpret_cast<uint4 *>(&table);
    for (int i = threadIdx.x; i < a.jump_digits * 32; i += kSampleThreads) dst[i] = src[i];
    __syncthreads();
    sample_thread<T>(a, out, (int64_t)blockIdx.x * kSampleThreads + threadIdx.x, (int64_t)gridDim.x * kSampleThreads,
                     table);
}

// ... the stream variant (space_sample.cuh): the generator comes from the record (or the override) and the last CTA
// to take a ticket writes the advanced state back, so one launch both reads and moves the stream
template <typename T>
__global__ void __launch_bounds__(kSampleThreads) space_sample_stream_kernel(const SampleArgs a, const SampleStream s,
                                                                             T *__restrict__ out) {
    __shared__ LcgJumpTable table;
    __shared__ Pcg64 start;
    const uint4 *src = reinterpret_cast<const uint4 *>(&kLcgJump);
    uint4 *dst = reinterpret_cast<uint4 *>(&table);
    for (int i = threadIdx.x; i < a.jump_digits * 32; i += kSampleThreads) dst[i] = src[i];
    if (threadIdx.x == 0) start = sample_stream_start(s);   // overlaps the table's loads
    __syncthreads();
    const Pcg64 g = start;
    // The ticket: this CTA's read of the record has returned (its value is in shared memory), so the last CTA to take
    // one writes after every read.  Its result is only needed after the draws, which hide the round trip.
    unsigned long long ticket = 0;
    if (threadIdx.x == 0) ticket = atomicAdd(reinterpret_cast<unsigned long long *>(s.record + 4), 1ULL);
    sample_thread<T>(a, g, a.hop_geo * g.inc, out, (int64_t)blockIdx.x * kSampleThreads + threadIdx.x,
                     (int64_t)gridDim.x * kSampleThreads, table);
    if (threadIdx.x == 0 && ticket == gridDim.x - 1ULL) sample_stream_finish(s, g);
}

// ---------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------
struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(int dev) {
        cudaGetDevice(&prev);
        if (prev != dev) cudaSetDevice(dev);
        else prev = -1;
    }
    ~DeviceGuard() {
        if (prev >= 0) cudaSetDevice(prev);
    }
};

// the device a caller-owned buffer lives on (these utilities take no handle)
static int device_of(const void *ptr) {
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, ptr) != cudaSuccess || at.type != cudaMemoryTypeDevice) {
        cudaGetLastError();
        return -1;
    }
    return at.device;
}

extern "C" int b200gym_create(const b200gym_config *cfg, int64_t num_envs, int device, b200gym_t **out) {
    if (!cfg || !out) return fail(nullptr, "b200gym_create: null argument");
    *out = nullptr;
    if (!kind_ok(cfg->kind)) return fail(nullptr, "b200gym_create: unknown env kind %d", cfg->kind);
    if ((cfg->kind == B200GYM_LUNARLANDER || cfg->kind == B200GYM_LUNARLANDER_CONT) &&
        !(-12.0 < cfg->param[0] && cfg->param[0] < 0.0))  // the assert of lunar_lander.py:210-212 (0.0 included: no
                                                          // silent default -- callers pass the reference's -10.0)
        return fail(nullptr, "b200gym_create: gravity (current value: %g) must be between -12 and 0", cfg->param[0]);
    if (num_envs <= 0) return fail(nullptr, "b200gym_create: num_envs must be positive (got %lld)", (long long)num_envs);
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        return fail(nullptr, "b200gym_create: no CUDA device available (%s); this engine has no CPU fallback",
                    cudaGetErrorString(e));
    if (device < 0 || device >= ndev) return fail(nullptr, "b200gym_create: bad device %d (have %d)", device, ndev);
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) == cudaSuccess && (prop.major != 9 || prop.minor != 0))
        return fail(nullptr, "b200gym_create: device %d is sm_%d%d; this library contains sm_90a code only",
                    device, prop.major, prop.minor);
    b200gym *h = new (std::nothrow) b200gym();
    if (!h) return fail(nullptr, "b200gym_create: out of host memory");
    h->cfg = *cfg;
    h->n = num_envs;
    h->device = device;
    h->S = k_state_dim[cfg->kind];
    h->D = k_obs_dim[cfg->kind];
    h->A = k_act_dim[cfg->kind];
    h->NACT = k_nact[cfg->kind];
    h->sm_count = prop.multiProcessorCount > 0 ? prop.multiProcessorCount : 132;
    {
        const char *kc = getenv("B200GYM_KERNEL");
        if (kc && (kc[0] == 'a' || kc[0] == 'p' || kc[0] == 'l' || kc[0] == 'b'))
            h->kernel_choice = kc[0] == 'a' ? 0 : kc[0] == 'b' ? 2 : 1;
        const char *pfb = getenv("B200GYM_P2P_FUSE_BARRIER");
        if (pfb && (pfb[0] == '0' || pfb[0] == '1')) h->p2p_fuse = pfb[0] - '0';
        const char *btd = getenv("B200GYM_BOX2D_TOI_DEFER");
        if (btd && (btd[0] == '0' || btd[0] == '1')) h->box2d_toi_defer = btd[0] - '0';
        const char *bdf = getenv("B200GYM_BOX2D_DEFER");
        if (bdf && (bdf[0] == '0' || bdf[0] == '1')) h->box2d_defer = bdf[0] - '0';
    }
    DeviceGuard guard(device);
    const size_t n = (size_t)num_envs;
    cudaError_t es[5] = {
        cudaMalloc(&h->state, sizeof(double) * n * (h->S > 0 ? h->S : 1)), cudaMalloc(&h->elapsed, sizeof(int32_t) * n),
        cudaMalloc(&h->flags, n), cudaMalloc(&h->rng, 32 * n), cudaMalloc(&h->invalid, sizeof(unsigned long long))};
    for (cudaError_t ei : es)
        if (ei != cudaSuccess) {
            fail(nullptr, "b200gym_create: cudaMalloc failed: %s", cudaGetErrorString(ei));
            b200gym_destroy(h);
            return 1;
        }
    if (cudaHostAlloc((void **)&h->invalid_seen, sizeof(unsigned long long), cudaHostAllocMapped) != cudaSuccess ||
        cudaHostGetDevicePointer((void **)&h->invalid_seen_dev, h->invalid_seen, 0) != cudaSuccess) {
        fail(nullptr, "b200gym_create: cannot allocate the mapped invalid-action flag: %s", cudaGetErrorString(cudaGetLastError()));
        b200gym_destroy(h);
        return 1;
    }
    *h->invalid_seen = 0ULL;
    h->is_lunar = cfg->kind == B200GYM_LUNARLANDER || cfg->kind == B200GYM_LUNARLANDER_CONT;
    h->is_walker = cfg->kind == B200GYM_BIPEDALWALKER || cfg->kind == B200GYM_BIPEDALWALKER_HARDCORE;
    if (h->is_lunar) {  // LunarLander.__init__ arguments (lunar_lander.py:194-233)
        h->lunar_opts.continuous = cfg->kind == B200GYM_LUNARLANDER_CONT;
        h->lunar_opts.wind = (cfg->flags & B200GYM_LUNAR_ENABLE_WIND) != 0;
        h->lunar_opts.gravity = (float)cfg->param[0];
        h->lunar_opts.wind_power = cfg->param[1];
        h->lunar_opts.turbulence_power = cfg->param[2];
    }
    if (h->is_lunar || h->is_walker) {
        const bool lun = h->is_lunar;
        const size_t words = lun ? lunar::kWords
                                 : (cfg->kind == B200GYM_BIPEDALWALKER_HARDCORE ? walker::kWordsHC : walker::kWords);
        if (cudaMalloc(&h->lunar_rec, sizeof(uint32_t) * words * n) != cudaSuccess ||
            cudaMemset(h->lunar_rec, 0, sizeof(uint32_t) * words * n) != cudaSuccess ||
            cudaMalloc((void **)&h->reset_list, sizeof(int32_t) * n) != cudaSuccess ||
            cudaMalloc((void **)&h->toi_list, sizeof(int32_t) * n) != cudaSuccess ||
            cudaMalloc((void **)&h->toi_count, sizeof(int32_t) * kResetSlots) != cudaSuccess ||
            cudaMemset(h->toi_count, 0, sizeof(int32_t) * kResetSlots) != cudaSuccess ||
            cudaMalloc((void **)&h->toi_mid, sizeof(uint32_t) * kToiMidWords * n) != cudaSuccess ||
            cudaMalloc((void **)&h->reset_count, sizeof(int32_t) * kResetSlots) != cudaSuccess ||
            cudaMemset(h->reset_count, 0, sizeof(int32_t) * kResetSlots) != cudaSuccess ||
            (lun ? lunar_upload_consts(h) : walker_upload_consts(h))) {
            fail(nullptr, "b200gym_create: Box2D-task state allocation failed");
            b200gym_destroy(h);
            return 1;
        }
    }
    const cudaError_t ms[5] = {cudaMemset(h->state, 0, sizeof(double) * n * (h->S > 0 ? h->S : 1)),
                               cudaMemset(h->elapsed, 0, sizeof(int32_t) * n), cudaMemset(h->flags, 0, n),
                               cudaMemset(h->rng, 0, 32 * n), cudaMemset(h->invalid, 0, sizeof(unsigned long long))};
    bool ms_ok = true;
    for (cudaError_t mi : ms) ms_ok = ms_ok && mi == cudaSuccess;
    if (!ms_ok || cudaDeviceSynchronize() != cudaSuccess) {
        fail(nullptr, "b200gym_create: device initialisation failed: %s", cudaGetErrorString(cudaGetLastError()));
        b200gym_destroy(h);
        return 1;
    }
    if (prepare_step(h)) {
        fail(nullptr, "b200gym_create: step kernel set-up failed: %s", b200gym_last_error(h));
        b200gym_destroy(h);
        return 1;
    }
    *out = h;
    return 0;
}

static void free_host_io(b200gym *h) {
    if (!h->host_ready) return;
    cudaFreeHost(h->hio.actions); cudaFreeHost(h->hio.obs); cudaFreeHost(h->hio.reward);
    cudaFreeHost(h->hio.terminated); cudaFreeHost(h->hio.truncated); cudaFreeHost(h->hio.final_obs);
    cudaFreeHost(h->h_invalid);
    cudaFree(h->dio.actions);
    cudaFree(h->d_mask);
    if (h->hevent) cudaEventDestroy(h->hevent);
    for (cudaStream_t st : h->hstream)
        if (st) cudaStreamDestroy(st);
    h->host_ready = false;
}

extern "C" void b200gym_destroy(b200gym_t *h) {
    if (!h) return;
    DeviceGuard guard(h->device);
    free_host_io(h);
    cudaFree(h->state);
    cudaFree(h->elapsed);
    cudaFree(h->flags);
    cudaFree(h->rng);
    cudaFree(h->invalid);
    if (h->invalid_seen) cudaFreeHost(h->invalid_seen);
    cudaFree(h->lunar_rec);
    cudaFree(h->reset_list);
    cudaFree(h->reset_count);
    cudaFree(h->toi_list);
    cudaFree(h->toi_count);
    cudaFree(h->toi_mid);
    if (h->snap_bad) cudaFreeHost(h->snap_bad);
    cudaFree(h->snap_scratch);
    if (h->from_batch) b200gym_destroy(h->from_batch);
    cudaFree(h->norm_rows);
    if (h->sub.final64) cudaFreeHost(h->sub.final64);
    if (h->sub.ep_r) cudaFreeHost(h->sub.ep_r);
    if (h->sub.ep_l) cudaFreeHost(h->sub.ep_l);
    cudaFree(h->sub.obs);
    cudaFree(h->sub.fin);
    cudaFree(h->sub.reward);
    cudaFree(h->sub.term);
    cudaFree(h->sub.trunc);
    cudaFree(h->sub.out);
    if (h->p2p.base) {
        for (int r = 0; r < h->p2p.world; r++)
            if (r != h->p2p.rank && h->p2p.peer[r]) cudaIpcCloseMemHandle(h->p2p.peer[r]);
        cudaFree(h->p2p.base);
        cudaFree(h->d_peer_flags);
        cudaFree(h->p2p_done);
    }
    delete h;
}

extern "C" int b200gym_seed_range(b200gym_t *h, const uint32_t base_words[4], int64_t first_index, void *stream) {
    if (!h || !base_words) return fail(h, "b200gym_seed_range: null argument");
    if (first_index < 0) return fail(h, "b200gym_seed_range: negative first_index");
    DeviceGuard guard(h->device);
    seed_range_kernel<<<blocks_for(h->n), kThreads, 0, (cudaStream_t)stream>>>(
        h->rng, h->n, base_words[0], base_words[1], base_words[2], base_words[3], (uint64_t)first_index);
    CK(h, cudaGetLastError());
    if (h->is_walker) {
        walker_clear_rng32_kernel<<<blocks_for(h->n), kThreads, 0, (cudaStream_t)stream>>>(h->lunar_rec, nullptr, h->n);
        CK(h, cudaGetLastError());
    }
    return 0;
}

extern "C" int b200gym_seed_each(b200gym_t *h, const uint32_t *ent_host, const uint8_t *mask_host, void *stream) {
    if (!h || !ent_host) return fail(h, "b200gym_seed_each: null argument");
    DeviceGuard guard(h->device);
    cudaStream_t st = (cudaStream_t)stream;
    uint32_t *d_ent = nullptr;
    uint8_t *d_mask = nullptr;
    CK(h, cudaMalloc(&d_ent, 16 * (size_t)h->n));
    cudaError_t e = cudaMemcpyAsync(d_ent, ent_host, 16 * (size_t)h->n, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess && mask_host) {
        e = cudaMalloc(&d_mask, (size_t)h->n);
        if (e == cudaSuccess) e = cudaMemcpyAsync(d_mask, mask_host, (size_t)h->n, cudaMemcpyHostToDevice, st);
    }
    if (e == cudaSuccess) {
        seed_each_kernel<<<blocks_for(h->n), kThreads, 0, st>>>(h->rng, h->n, d_ent, d_mask);
        if (h->is_walker)
            walker_clear_rng32_kernel<<<blocks_for(h->n), kThreads, 0, st>>>(h->lunar_rec, d_mask, h->n);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    cudaFree(d_ent);
    cudaFree(d_mask);
    if (e != cudaSuccess) return fail(h, "b200gym_seed_each: %s", cudaGetErrorString(e));
    return 0;
}

extern "C" int b200gym_reset(b200gym_t *h, const uint8_t *mask_dev, const double *bounds_host, float *obs_dev,
                             void *stream) {
    if (!h) return fail(h, "b200gym_reset: null handle");
    DeviceGuard guard(h->device);
    return launch_reset(h, mask_dev, bounds_host, obs_dev, (cudaStream_t)stream);
}

static StepArgs make_args(b200gym *h, const void *actions, float *obs, double *reward, uint8_t *term,
                          uint8_t *trunc, float *final_obs) {
    StepArgs a;
    a.state = h->state; a.elapsed = h->elapsed; a.flags = h->flags; a.rng = h->rng; a.invalid = h->invalid;
    a.invalid_seen = h->invalid_seen_dev;
    a.lunar_rec = h->lunar_rec;
    a.actions = actions; a.obs = obs; a.reward = reward; a.terminated = term; a.truncated = trunc;
    a.final_obs = final_obs;
    a.n = h->n; a.first = 0; a.count = h->n;
    a.max_steps = h->cfg.max_episode_steps; a.autoreset = h->cfg.autoreset; a.param0 = h->cfg.param[0];
    a.lunar_opts = h->lunar_opts;
    a.reset_list = nullptr; a.reset_count = nullptr;
    a.toi_list = nullptr; a.toi_count = nullptr; a.toi_mid = nullptr;
    a.p2p_done = nullptr; a.p2p_peer_flags = nullptr; a.p2p_my_flags = nullptr; a.p2p_timed_out = nullptr;
    a.p2p_step = 0; a.p2p_timeout_ns = 0; a.p2p_world = 0; a.p2p_rank = 0;
    a.npeer = 0;
    a.bulk_sink = 0;
    return a;
}

extern "C" int b200gym_step(b200gym_t *h, const void *actions_dev, int action_dtype, float *obs_dev,
                            double *reward_dev, uint8_t *terminated_dev, uint8_t *truncated_dev,
                            float *final_obs_dev, void *stream) {
    if (!h) return fail(h, "b200gym_step: null handle");
    if (!actions_dev || !obs_dev || !reward_dev || !terminated_dev || !truncated_dev)
        return fail(h, "b200gym_step: null buffer");
    DeviceGuard guard(h->device);
    const StepArgs a = make_args(h, actions_dev, obs_dev, reward_dev, terminated_dev, truncated_dev, final_obs_dev);
    return launch_step(h, a, action_dtype, (cudaStream_t)stream);
}

extern "C" int b200gym_rollout(b200gym_t *h, const void *actions_dev, int action_dtype, int32_t T, float *obs_dev,
                               double *reward_dev, uint8_t *terminated_dev, uint8_t *truncated_dev, float *final_obs_dev,
                               float *last_obs_dev, void *stream) {
    if (!h) return fail(h, "b200gym_rollout: null handle");
    if (T < 1) return fail(h, "b200gym_rollout: T must be at least 1 (got %d)", T);
    if (!actions_dev || !obs_dev || !reward_dev || !terminated_dev || !truncated_dev || !last_obs_dev)
        return fail(h, "b200gym_rollout: null buffer");
    DeviceGuard guard(h->device);
    const StepArgs a = make_args(h, actions_dev, obs_dev, reward_dev, terminated_dev, truncated_dev, final_obs_dev);
    return launch_rollout(h, a, action_dtype, T, last_obs_dev, (cudaStream_t)stream);
}

extern "C" int b200gym_invalid_actions(b200gym_t *h, void *stream, int64_t *count_out) {
    if (!h || !count_out) return fail(h, "b200gym_invalid_actions: null argument");
    DeviceGuard guard(h->device);
    cudaStream_t st = (cudaStream_t)stream;
    unsigned long long v = 0;
    CK(h, cudaMemcpyAsync(&v, h->invalid, sizeof v, cudaMemcpyDeviceToHost, st));
    CK(h, cudaMemsetAsync(h->invalid, 0, sizeof v, st));
    CK(h, cudaStreamSynchronize(st));
    *h->invalid_seen = 0ULL;
    *count_out = (int64_t)v;
    return 0;
}

extern "C" int b200gym_invalid_seen(const b200gym_t *h) {
    if (!h || !h->invalid_seen) return -1;
    return *reinterpret_cast<volatile unsigned long long *>(h->invalid_seen) != 0ULL ? 1 : 0;
}

extern "C" int b200gym_selftest_trig(const double *x_dev, int64_t n, double *sin_dev, double *cos_dev, double *sq_dev,
                                     void *stream) {
    if (!x_dev || !sin_dev || !cos_dev || n <= 0) return fail(nullptr, "b200gym_selftest_trig: bad argument");
    const int dev = device_of(x_dev);
    if (dev < 0) return fail(nullptr, "b200gym_selftest_trig: x is not a device pointer");
    DeviceGuard guard(dev);
    selftest_trig_kernel<<<blocks_for(n), kThreads, 0, (cudaStream_t)stream>>>(x_dev, n, sin_dev, cos_dev, sq_dev);
    CK(nullptr, cudaGetLastError());
    return 0;
}

extern "C" int b200gym_selftest_tanh(const float *x_dev, int64_t n, float *y_dev, void *stream) {
    if (!x_dev || !y_dev || n <= 0) return fail(nullptr, "b200gym_selftest_tanh: bad argument");
    const int dev = device_of(x_dev);
    if (dev < 0) return fail(nullptr, "b200gym_selftest_tanh: x is not a device pointer");
    DeviceGuard guard(dev);
    selftest_tanh_kernel<<<blocks_for(n), kThreads, 0, (cudaStream_t)stream>>>(x_dev, n, y_dev);
    CK(nullptr, cudaGetLastError());
    return 0;
}

extern "C" int b200gym_selftest_exp(const float *x_dev, int64_t n, float *y_dev, void *stream) {
    if (!x_dev || !y_dev || n <= 0) return fail(nullptr, "b200gym_selftest_exp: bad argument");
    const int dev = device_of(x_dev);
    if (dev < 0) return fail(nullptr, "b200gym_selftest_exp: x is not a device pointer");
    DeviceGuard guard(dev);
    selftest_exp_kernel<<<blocks_for(n), kThreads, 0, (cudaStream_t)stream>>>(x_dev, n, y_dev);
    CK(nullptr, cudaGetLastError());
    return 0;
}

// b2probe.cu: the probe kernel, in a module of its own so that this module's kernels compile as they did without it
cudaError_t b2probe_launch(int op, const float *in_dev, int64_t n, float *out_dev, cudaStream_t stream);
int b2probe_num_ops();

extern "C" int b200gym_selftest_box2d(int op, const float *in_dev, int64_t n, float *out_dev, void *stream) {
    if (op < 0 || op >= b2probe_num_ops() || !in_dev || !out_dev || n <= 0)
        return fail(nullptr, "b200gym_selftest_box2d: bad argument");
    const int dev = device_of(in_dev);
    if (dev < 0 || device_of(out_dev) != dev) return fail(nullptr, "b200gym_selftest_box2d: buffers are not on one device");
    DeviceGuard guard(dev);
    CK(nullptr, b2probe_launch(op, in_dev, n, out_dev, (cudaStream_t)stream));
    return 0;
}

extern "C" int b200gym_box2d_overflows(b200gym_t *h, void *stream, int64_t *count_out) {
    if (!h || !count_out) return fail(h, "b200gym_box2d_overflows: null argument");
    if (!h->is_lunar && !h->is_walker) return fail(h, "b200gym_box2d_overflows: not a Box2D-task handle");
    DeviceGuard guard(h->device);
    cudaStream_t st = (cudaStream_t)stream;
    unsigned long long *d = nullptr, v = 0;
    CK(h, cudaMalloc((void **)&d, sizeof *d));
    cudaError_t e = cudaMemsetAsync(d, 0, sizeof *d, st);
    if (e == cudaSuccess) {
        const int64_t row = h->is_lunar ? lunar::W_FLAGS : walker::W_FLAGS;
        box2d_overflow_kernel<<<blocks_for(h->n), kThreads, 0, st>>>(h->lunar_rec + row * h->n, h->n, d);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(&v, d, sizeof v, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    cudaFree(d);
    if (e != cudaSuccess) return fail(h, "b200gym_box2d_overflows: %s", cudaGetErrorString(e));
    *count_out = (int64_t)v;
    return 0;
}

extern "C" int b200gym_box2d_list_counts(b200gym_t *h, void *stream, int slots, int32_t *parked_out, int32_t *resets_out) {
    if (!h || !parked_out || !resets_out) return fail(h, "b200gym_box2d_list_counts: null argument");
    if (!h->is_lunar && !h->is_walker) return fail(h, "b200gym_box2d_list_counts: not a Box2D-task handle");
    if (slots < 1 || slots > kResetSlots)
        return fail(h, "b200gym_box2d_list_counts: slots must be in [1, %d], got %d", kResetSlots, slots);
    DeviceGuard guard(h->device);
    cudaStream_t st = (cudaStream_t)stream;
    const size_t bytes = sizeof(int32_t) * (size_t)slots;
    cudaError_t e = cudaMemcpyAsync(parked_out, h->toi_count, bytes, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(resets_out, h->reset_count, bytes, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return fail(h, "b200gym_box2d_list_counts: %s", cudaGetErrorString(e));
    return 0;
}

extern "C" int b200gym_selftest(int device, int64_t samples, uint64_t seed, int64_t *mismatches_out) {
    if (!mismatches_out || samples <= 0) return fail(nullptr, "b200gym_selftest: bad argument");
    DeviceGuard guard(device);
    unsigned long long *d = nullptr;
    if (cudaMalloc(&d, sizeof *d) != cudaSuccess) return fail(nullptr, "b200gym_selftest: cudaMalloc failed");
    cudaMemset(d, 0, sizeof *d);
    selftest_div_kernel<<<blocks_for(samples), kThreads>>>(samples, seed, d);
    unsigned long long v = 0;
    cudaError_t e = cudaMemcpy(&v, d, sizeof v, cudaMemcpyDeviceToHost);
    cudaFree(d);
    if (e != cudaSuccess) return fail(nullptr, "b200gym_selftest: %s", cudaGetErrorString(e));
    *mismatches_out = (int64_t)v;
    return 0;
}

// ---- fused all-gather over NVLink peer memory ----------------------------------------------
static size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

extern "C" int b200gym_p2p_create(b200gym_t *h, int world, int rank, void *ipc_handle_out /*64 B*/,
                                  b200gym_p2p_layout *layout_out) {
    if (!h || !ipc_handle_out || !layout_out) return fail(h, "b200gym_p2p_create: null argument");
    if (world < 1 || world > B200GYM_MAX_PEERS + 1 || rank < 0 || rank >= world)
        return fail(h, "b200gym_p2p_create: bad world/rank %d/%d (at most %d ranks)", world, rank, B200GYM_MAX_PEERS + 1);
    if (h->p2p.base) return fail(h, "b200gym_p2p_create: already created");
    DeviceGuard guard(h->device);
    auto &P = h->p2p;
    const size_t rows = (size_t)world * (size_t)h->n;
    P.world = world;
    P.rank = rank;
    P.off_obs = 0;
    P.off_reward = align_up(P.off_obs + rows * h->D * sizeof(float), 256);
    P.off_term = align_up(P.off_reward + rows * sizeof(double), 256);
    P.off_trunc = align_up(P.off_term + rows, 256);
    P.set_bytes = align_up(P.off_trunc + rows, 256);
    P.off_flags = 2 * P.set_bytes;          // [0,64): one uint64 step counter per rank; [128,132): sticky time-out word
    P.bytes = P.off_flags + 256;
    if (const char *ts = getenv("B200GYM_P2P_TIMEOUT_S")) {
        const double v = atof(ts);
        if (v > 0.0) P.timeout_ns = (unsigned long long)(v * 1e9);
    }
    CK(h, cudaMalloc((void **)&P.base, P.bytes));
    CK(h, cudaMemset(P.base, 0, P.bytes));
    CK(h, cudaDeviceSynchronize());
    cudaIpcMemHandle_t ipc;
    CK(h, cudaIpcGetMemHandle(&ipc, P.base));
    static_assert(sizeof(ipc) == 64, "cudaIpcMemHandle_t is 64 bytes");
    memcpy(ipc_handle_out, &ipc, sizeof ipc);
    layout_out->base = P.base;
    layout_out->set_bytes = P.set_bytes;
    layout_out->off_obs = P.off_obs;
    layout_out->off_reward = P.off_reward;
    layout_out->off_terminated = P.off_term;
    layout_out->off_truncated = P.off_trunc;
    layout_out->rows = (int64_t)rows;
    return 0;
}

extern "C" int b200gym_p2p_connect(b200gym_t *h, const void *all_ipc_handles /*world x 64 B*/) {
    if (!h || !all_ipc_handles) return fail(h, "b200gym_p2p_connect: null argument");
    auto &P = h->p2p;
    if (!P.base) return fail(h, "b200gym_p2p_connect: call b200gym_p2p_create first");
    if (P.connected) return 0;
    DeviceGuard guard(h->device);
    for (int r = 0; r < P.world; r++) {
        if (r == P.rank) {
            P.peer[r] = P.base;
            continue;
        }
        cudaIpcMemHandle_t ipc;
        memcpy(&ipc, (const char *)all_ipc_handles + 64 * r, sizeof ipc);
        void *ptr = nullptr;
        CK(h, cudaIpcOpenMemHandle(&ptr, ipc, cudaIpcMemLazyEnablePeerAccess));
        P.peer[r] = (unsigned char *)ptr;
    }
    P.connected = true;
    return 0;
}

extern "C" int b200gym_step_p2p(b200gym_t *h, const void *actions_dev, int action_dtype, float *final_obs_dev,
                                void *stream, int *set_out) {
    if (!h || !actions_dev) return fail(h, "b200gym_step_p2p: null argument");
    auto &P = h->p2p;
    if (!P.connected) return fail(h, "b200gym_step_p2p: peers are not connected");
    DeviceGuard guard(h->device);
    cudaStream_t st = (cudaStream_t)stream;
    P.step += 1;
    const int set = (int)(P.step & 1);
    const size_t row0 = (size_t)P.rank * (size_t)h->n;
    auto obs_of = [&](unsigned char *b) { return (float *)(b + set * P.set_bytes + P.off_obs) + row0 * h->D; };
    auto rew_of = [&](unsigned char *b) { return (double *)(b + set * P.set_bytes + P.off_reward) + row0; };
    auto term_of = [&](unsigned char *b) { return (uint8_t *)(b + set * P.set_bytes + P.off_term) + row0; };
    auto trunc_of = [&](unsigned char *b) { return (uint8_t *)(b + set * P.set_bytes + P.off_trunc) + row0; };
    StepArgs a = make_args(h, actions_dev, obs_of(P.base), rew_of(P.base), term_of(P.base), trunc_of(P.base),
                           final_obs_dev);
    int np = 0;
    for (int r = 0; r < P.world; r++) {
        if (r == P.rank) continue;
        a.peer_obs[np] = obs_of(P.peer[r]);
        a.peer_reward[np] = rew_of(P.peer[r]);
        a.peer_term[np] = term_of(P.peer[r]);
        a.peer_trunc[np] = trunc_of(P.peer[r]);
        np++;
    }
    a.npeer = np;
    if (P.world > 1 && !h->d_peer_flags) {
        unsigned long long *pf[B200GYM_MAX_PEERS + 1];
        for (int r = 0; r < P.world; r++) pf[r] = (unsigned long long *)(P.peer[r] + P.off_flags);
        CK(h, cudaMalloc((void **)&h->d_peer_flags, sizeof pf));
        CK(h, cudaMemcpy(h->d_peer_flags, pf, sizeof pf, cudaMemcpyHostToDevice));
        CK(h, cudaMalloc((void **)&h->p2p_done, sizeof(unsigned int)));
        CK(h, cudaMemset(h->p2p_done, 0, sizeof(unsigned int)));
    }
    if (P.world > 1 && h->p2p_fuse) {   // offer kernel G the step barrier (it takes it when it covers the whole range)
        a.p2p_done = h->p2p_done;
        a.p2p_peer_flags = h->d_peer_flags;
        a.p2p_my_flags = (const unsigned long long *)(P.base + P.off_flags);
        a.p2p_timed_out = (int *)(P.base + P.off_flags + 128);
        a.p2p_step = P.step; a.p2p_timeout_ns = P.timeout_ns; a.p2p_world = P.world; a.p2p_rank = P.rank;
    }
    h->p2p_barrier_fused = false;
    if (launch_step(h, a, action_dtype, st)) return 1;
    if (P.world > 1 && !h->p2p_barrier_fused) {
        // tell every peer that my rows of step `P.step` are in its buffers, then wait for theirs
        p2p_sync_kernel<<<1, 32, 0, st>>>(h->d_peer_flags, (const unsigned long long *)(P.base + P.off_flags), P.world,
                                          P.rank, P.step, P.timeout_ns, (int *)(P.base + P.off_flags + 128));
        CK(h, cudaGetLastError());
    }
    if (set_out) *set_out = set;
    return 0;
}

extern "C" int b200gym_p2p_status(b200gym_t *h, void *stream, int *timed_out_peer) {
    if (!h || !timed_out_peer) return fail(h, "b200gym_p2p_status: null argument");
    auto &P = h->p2p;
    if (!P.base) return fail(h, "b200gym_p2p_status: no gather allocation");
    DeviceGuard guard(h->device);
    int v = 0;
    CK(h, cudaMemcpyAsync(&v, P.base + P.off_flags + 128, sizeof v, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
    CK(h, cudaStreamSynchronize((cudaStream_t)stream));
    *timed_out_peer = v - 1;   // -1: every step barrier completed
    if (v) return fail(h, "b200gym_step_p2p: rank %d did not deliver its rows within %.0f s (peer lost?)", v - 1,
                       (double)P.timeout_ns * 1e-9);
    return 0;
}

// ---- stateless device utilities for the vector-aware wrappers (SURVEY.md 8f) -----------------------
extern "C" int b200gym_episode_stats(const double *reward_dev, const uint8_t *terminated_dev, const uint8_t *truncated_dev,
                                     float *return_acc_dev, int32_t *length_acc_dev, float *episode_r_dev,
                                     int32_t *episode_l_dev, uint8_t *episode_mask_dev, uint64_t *ring_dev,
                                     uint64_t *counter_dev, int ring_size, int64_t n, void *stream) {
    if (!reward_dev || !terminated_dev || !truncated_dev || !return_acc_dev || !length_acc_dev || !episode_r_dev ||
        !episode_l_dev || !episode_mask_dev || !counter_dev || n <= 0 || (ring_size > 0 && !ring_dev))
        return fail(nullptr, "b200gym_episode_stats: bad argument");
    const int dev = device_of(reward_dev);
    if (dev < 0) return fail(nullptr, "b200gym_episode_stats: reward is not a device pointer");
    DeviceGuard guard(dev);
    episode_stats_kernel<<<blocks_for(n), kThreads, 0, (cudaStream_t)stream>>>(
        reward_dev, terminated_dev, truncated_dev, return_acc_dev, length_acc_dev, episode_r_dev, episode_l_dev,
        episode_mask_dev, (unsigned long long *)ring_dev, (unsigned long long *)counter_dev, ring_size, n);
    CK(nullptr, cudaGetLastError());
    return 0;
}

static int norm_dims_ok(int dim) { return dim == 1 || dim == 2 || dim == 3 || dim == 4 || dim == 6 || dim == 8 || dim == 24; }

static unsigned norm_grid(int64_t total, int block) {
    int64_t g = (total + block - 1) / block;
    if (g > kNormMaxCtas) g = kNormMaxCtas;       // 132 SMs x 8: one resident wave, grid-stride beyond
    return (unsigned)(g < 1 ? 1 : g);
}

extern "C" int b200gym_rms_moments(const void *x_dev, int is_f64, int64_t n, int dim, const double *stats_dev,
                                   double *scratch_dev, double *work_dev, void *stream) {
    if (!x_dev || !stats_dev || !scratch_dev || !work_dev || n <= 0 || !norm_dims_ok(dim))
        return fail(nullptr, "b200gym_rms_moments: bad argument (dim must be one of 1, 2, 3, 4, 6, 8, 24)");
    const int dev = device_of(x_dev);
    if (dev < 0) return fail(nullptr, "b200gym_rms_moments: x is not a device pointer");
    DeviceGuard guard(dev);
    const int block = (dim == 3 || dim == 6 || dim == 24) ? 192 : 256;
    const int64_t total = n * dim;
    cudaStream_t st = (cudaStream_t)stream;
    if (is_f64)
        rms_moments_kernel<double, false><<<norm_grid(total, block), block, 0, st>>>(
            (const double *)x_dev, nullptr, nullptr, 0.0, total, dim, stats_dev, scratch_dev, work_dev);
    else
        rms_moments_kernel<float, false><<<norm_grid(total, block), block, 0, st>>>(
            (const float *)x_dev, nullptr, nullptr, 0.0, total, dim, stats_dev, scratch_dev, work_dev);
    CK(nullptr, cudaGetLastError());
    return 0;
}

extern "C" int b200gym_return_moments(double *returns_dev, const double *reward_dev, double gamma, int64_t n,
                                      const double *stats_dev, double *scratch_dev, double *work_dev, void *stream) {
    if (!returns_dev || !reward_dev || !stats_dev || !scratch_dev || !work_dev || n <= 0)
        return fail(nullptr, "b200gym_return_moments: bad argument");
    const int dev = device_of(returns_dev);
    if (dev < 0) return fail(nullptr, "b200gym_return_moments: returns is not a device pointer");
    DeviceGuard guard(dev);
    rms_moments_kernel<double, true><<<norm_grid(n, 256), 256, 0, (cudaStream_t)stream>>>(
        nullptr, returns_dev, reward_dev, gamma, n, 1, stats_dev, scratch_dev, work_dev);
    CK(nullptr, cudaGetLastError());
    return 0;
}

extern "C" int b200gym_rms_apply_obs(const float *obs_dev, float *out_dev, int64_t n, int dim, const double *stats_dev,
                                     double *stats_next_dev, const double *scratch_dev, double *scratch_next_dev,
                                     double batch_count, double epsilon, int update, void *stream) {
    if (!obs_dev || !out_dev || !stats_dev || !stats_next_dev || !scratch_dev || !scratch_next_dev || n <= 0 ||
        !norm_dims_ok(dim))
        return fail(nullptr, "b200gym_rms_apply_obs: bad argument (dim must be one of 1, 2, 3, 4, 6, 8, 24)");
    const int dev = device_of(obs_dev);
    if (dev < 0) return fail(nullptr, "b200gym_rms_apply_obs: obs is not a device pointer");
    DeviceGuard guard(dev);
    const int block = (dim == 3 || dim == 6 || dim == 24) ? 192 : 256;
    rms_apply_kernel<false><<<norm_grid(n * dim, block), block, 0, (cudaStream_t)stream>>>(
        obs_dev, out_dev, nullptr, nullptr, nullptr, nullptr, nullptr, n * dim, dim, stats_dev, stats_next_dev, scratch_dev,
        scratch_next_dev, batch_count, epsilon, update);
    CK(nullptr, cudaGetLastError());
    return 0;
}

extern "C" int b200gym_rms_apply_reward(const double *reward_dev, double *out_dev, double *returns_dev,
                                        const uint8_t *terminated_dev, const uint8_t *truncated_dev, int64_t n,
                                        const double *stats_dev, double *stats_next_dev, const double *scratch_dev,
                                        double *scratch_next_dev, double batch_count, double epsilon, void *stream) {
    if (!reward_dev || !out_dev || !returns_dev || !terminated_dev || !truncated_dev || !stats_dev || !stats_next_dev ||
        !scratch_dev || !scratch_next_dev || n <= 0)
        return fail(nullptr, "b200gym_rms_apply_reward: bad argument");
    const int dev = device_of(reward_dev);
    if (dev < 0) return fail(nullptr, "b200gym_rms_apply_reward: reward is not a device pointer");
    DeviceGuard guard(dev);
    rms_apply_kernel<true><<<norm_grid(n, 256), 256, 0, (cudaStream_t)stream>>>(
        nullptr, nullptr, reward_dev, out_dev, returns_dev, terminated_dev, truncated_dev, n, 1, stats_dev, stats_next_dev,
        scratch_dev, scratch_next_dev, batch_count, epsilon, 1);
    CK(nullptr, cudaGetLastError());
    return 0;
}

// the arguments both sampling entry points share; `what` names the caller in the error
static int sample_prepare(const char *what, int64_t rows, int cols, int64_t n_choices, const double *low_host,
                          const double *high_host, void *out_dev, SampleArgs &a, int &dev) {
    if (!out_dev || rows <= 0 || cols <= 0 || cols > kSampleMaxCols || n_choices < 0 || (n_choices > 0 && cols != 1) ||
        (n_choices == 0 && (!low_host || !high_host)) || rows > INT64_MAX / kSampleMaxCols)
        return fail(nullptr, "%s: bad argument (MultiDiscrete needs cols = 1, a Box 1 <= cols <= %d and its bounds)", what,
                    kSampleMaxCols);
    if ((uintptr_t)out_dev % 16) return fail(nullptr, "%s: out is not 16-byte aligned", what);
    a = SampleArgs{};
    a.total = rows * cols;
    a.cols = cols;
    a.n_choices = (double)n_choices;
    if (n_choices == 0) {
        for (int c = 0; c < cols; c++) {
            a.low[c] = low_host[c];
            a.high[c] = high_host[c];
            if (!std::isfinite(a.low[c]) || !std::isfinite(a.high[c]) || !std::isfinite(a.high[c] - a.low[c]))
                return fail(nullptr, "%s: column %d is not a bounded Box (low %g, high %g)", what, c, a.low[c], a.high[c]);
        }
    }
    dev = device_of(out_dev);
    if (dev < 0) return fail(nullptr, "%s: out is not a device pointer", what);
    return 0;
}

extern "C" int b200gym_sample_space(const uint64_t pcg64[4], int64_t rows, int cols, int64_t n_choices,
                                    const double *low_host, const double *high_host, void *out_dev, void *stream) {
    SampleArgs a;
    int dev;
    if (!pcg64) return fail(nullptr, "b200gym_sample_space: bad argument (null generator)");
    if (sample_prepare("b200gym_sample_space", rows, cols, n_choices, low_host, high_host, out_dev, a, dev)) return 1;
    a.start.state = make_u128(pcg64[0], pcg64[1]);
    a.start.inc = make_u128(pcg64[2], pcg64[3]);
    DeviceGuard guard(dev);
    const int vec = n_choices > 0 ? 2 : 4;
    const int64_t blocks = sample_blocks(a.total, vec);
    sample_setup(a, blocks * kSampleThreads, vec);
    cudaStream_t st = (cudaStream_t)stream;
    if (n_choices > 0)
        space_sample_kernel<long long><<<(unsigned)blocks, kSampleThreads, 0, st>>>(a, (long long *)out_dev);
    else
        space_sample_kernel<float><<<(unsigned)blocks, kSampleThreads, 0, st>>>(a, (float *)out_dev);
    CK(nullptr, cudaGetLastError());
    return 0;
}

extern "C" int b200gym_sample_space_stream(uint64_t *record_dev, const uint64_t override_pcg64[4], int64_t rows, int cols,
                                           int64_t n_choices, const double *low_host, const double *high_host,
                                           void *out_dev, void *stream) {
    SampleArgs a;
    int dev;
    if (!record_dev || (uintptr_t)record_dev % 16)
        return fail(nullptr, "b200gym_sample_space_stream: the record must be a 16-byte aligned device buffer");
    if (sample_prepare("b200gym_sample_space_stream", rows, cols, n_choices, low_host, high_host, out_dev, a, dev))
        return 1;
    if (device_of(record_dev) != dev)
        return fail(nullptr, "b200gym_sample_space_stream: the record is not on the device of out");
    SampleStream s{};
    s.record = record_dev;
    if (override_pcg64) {
        s.use_override = 1;
        for (int k = 0; k < 4; k++) s.override_words[k] = override_pcg64[k];
    }
    s.advance = lcg_jump_map((u128)a.total);
    DeviceGuard guard(dev);
    const int vec = n_choices > 0 ? 2 : 4;
    const int64_t blocks = sample_blocks(a.total, vec);
    sample_setup(a, blocks * kSampleThreads, vec);   // a.start is unused: the hop_plus it derives is recomputed on the device
    cudaStream_t st = (cudaStream_t)stream;
    if (n_choices > 0)
        space_sample_stream_kernel<long long><<<(unsigned)blocks, kSampleThreads, 0, st>>>(a, s, (long long *)out_dev);
    else
        space_sample_stream_kernel<float><<<(unsigned)blocks, kSampleThreads, 0, st>>>(a, s, (float *)out_dev);
    CK(nullptr, cudaGetLastError());
    return 0;
}

// ---- rollouts of random actions (b200gym_rollout_sampled) ----
template <int KIND>
static int launch_rollout_sampled_kind(b200gym *h, const StepArgs &a, int32_t T, float *last_obs, const RolloutDraws &d,
                                       const SampleStream &s, cudaStream_t st) {
    rollout_sampled_kernel<KIND><<<blocks_for(h->n), kThreads, 0, st>>>(a, T, last_obs, d, s);
    CK(h, cudaGetLastError());
    return 0;
}

extern "C" int b200gym_rollout_sampled(b200gym_t *h, uint64_t *record_dev, const uint64_t override_pcg64[4],
                                       int64_t n_choices, const double *low_host, const double *high_host, int32_t T,
                                       void *actions_out_dev, float *obs_dev, double *reward_dev,
                                       uint8_t *terminated_dev, uint8_t *truncated_dev, float *final_obs_dev,
                                       float *last_obs_dev, void *stream) {
    if (!h) return fail(h, "b200gym_rollout_sampled: null handle");
    if (T < 1) return fail(h, "b200gym_rollout_sampled: T must be at least 1 (got %d)", T);
    if (!record_dev || !actions_out_dev || !obs_dev || !reward_dev || !terminated_dev || !truncated_dev || !last_obs_dev)
        return fail(h, "b200gym_rollout_sampled: null buffer");
    if ((uintptr_t)record_dev % 16)
        return fail(h, "b200gym_rollout_sampled: the record must be a 16-byte aligned device buffer");
    if ((n_choices > 0) != (h->A == 0))
        return fail(h, "b200gym_rollout_sampled: %s", h->A == 0 ? "a Discrete env needs n_choices >= 1"
                                                                : "a Box env needs n_choices = 0 and its bounds");
    const int cols = std::max(h->A, 1);
    const int64_t draws_n = (int64_t)T * h->n;   // rows of the [T][n][cols] action output
    SampleArgs sa;
    int dev;
    if (sample_prepare("b200gym_rollout_sampled", draws_n, cols, n_choices, low_host, high_host, actions_out_dev, sa,
                       dev))
        return fail(h, "%s", b200gym_last_error(nullptr));
    if (dev != h->device || device_of(record_dev) != h->device)
        return fail(h, "b200gym_rollout_sampled: the record and the action output must be on the handle's device %d",
                    h->device);
    DeviceGuard guard(h->device);
    const StepArgs a = make_args(h, actions_out_dev, obs_dev, reward_dev, terminated_dev, truncated_dev, final_obs_dev);
    cudaStream_t st = (cudaStream_t)stream;
    if (h->is_lunar || h->is_walker) {
        // T consecutive sample() calls are T * n * cols consecutive draws in C order, which is the [T][n][cols] layout:
        // one sampling launch fills every slice, then the Box2D rollout steps through them
        if (b200gym_sample_space_stream(record_dev, override_pcg64, draws_n, cols, n_choices, low_host, high_host,
                                        actions_out_dev, stream))
            return fail(h, "%s", b200gym_last_error(nullptr));
        return launch_rollout_box2d(h, a, h->A == 0 ? B200GYM_ACT_I64 : B200GYM_ACT_F32, T, last_obs_dev, st);
    }
    SampleStream s{};
    s.record = record_dev;
    if (override_pcg64) {
        s.use_override = 1;
        for (int k = 0; k < 4; k++) s.override_words[k] = override_pcg64[k];
    }
    s.advance = lcg_jump_map((u128)sa.total);
    const LcgMap hop = lcg_jump_map((u128)(h->n - 1));
    RolloutDraws d{hop.mult, hop.geo, n_choices > 0 ? (double)n_choices : sa.low[0], n_choices > 0 ? 0.0 : sa.high[0], 0};
    for (uint64_t last = (uint64_t)(h->n - 1); last != 0; last >>= 4) d.jump_digits++;
    switch (h->cfg.kind) {
    case B200GYM_CARTPOLE: return launch_rollout_sampled_kind<B200GYM_CARTPOLE>(h, a, T, last_obs_dev, d, s, st);
    case B200GYM_MOUNTAINCAR: return launch_rollout_sampled_kind<B200GYM_MOUNTAINCAR>(h, a, T, last_obs_dev, d, s, st);
    case B200GYM_MOUNTAINCAR_CONT:
        return launch_rollout_sampled_kind<B200GYM_MOUNTAINCAR_CONT>(h, a, T, last_obs_dev, d, s, st);
    case B200GYM_PENDULUM: return launch_rollout_sampled_kind<B200GYM_PENDULUM>(h, a, T, last_obs_dev, d, s, st);
    case B200GYM_ACROBOT: return launch_rollout_sampled_kind<B200GYM_ACROBOT>(h, a, T, last_obs_dev, d, s, st);
    }
    return fail(h, "bad kind %d", h->cfg.kind);
}

// ---- closed-loop rollouts of a linear policy (b200gym_rollout_linear) ----
template <int KIND>
static int launch_rollout_linear_kind(b200gym *h, const StepArgs &a, int32_t T, float *last_obs,
                                      const LinearPolicyArgs &p, bool summary, cudaStream_t st) {
    if (summary) rollout_linear_kernel<KIND, true><<<blocks_for(h->n), kThreads, 0, st>>>(a, T, last_obs, p);
    else rollout_linear_kernel<KIND, false><<<blocks_for(h->n), kThreads, 0, st>>>(a, T, last_obs, p);
    CK(h, cudaGetLastError());
    return 0;
}

// A Box2D closed-loop rollout: per step, one launch of `policy` (linear_policy_kernel, mlp_policy_kernel,
// mlp_noisy_policy_kernel) with the arguments args_at(t) from the observation rows of the step before (first_obs for
// step 0), with `smem` bytes of dynamic shared memory, then launch_step_box2d into slice t.  Summary mode: every step
// runs in one scratch slice, and the policy launch of step t + 1 (or one last launch, with args_at(T - 1)) folds step t
// into the summary.  kernel / entry: names for the error messages.  hook(t, obs_in, s, after): launches of the
// caller's own around step t, made before the policy launch (after false, obs_in the policy's input) and after the
// step sequence (after true, s the step's outputs); non-zero fails the rollout.  input(obs): the rows the policy and
// the hook read in place of the observation rows obs of step t, made by launches of the caller's own before both;
// nullptr fails the rollout
struct NoStepHook {
    int operator()(int32_t, const float *, const StepArgs &, bool) const { return 0; }
};
struct RawStepInput {
    const float *operator()(const float *obs) const { return obs; }
};

template <typename Args, typename ArgsAt, typename Hook = NoStepHook, typename Input = RawStepInput>
static int launch_rollout_policy_box2d(b200gym *h, const StepArgs &a, int32_t T, float *last_obs,
                                       const float *first_obs, const ArgsAt &args_at,
                                       void (*policy)(const float *, void *, const Args, const double *,
                                                      const uint8_t *, const uint8_t *, int64_t, int32_t, int, int),
                                       size_t smem, bool summary, cudaStream_t st, const char *kernel,
                                       const char *entry, const Hook &hook = Hook{}, const Input &input = Input{}) {
    const int64_t n = h->n, D = h->D, cols = std::max(h->A, 1);
    const size_t act_row = (size_t)n * cols * (h->A == 0 ? sizeof(long long) : sizeof(float));
    const int action_dtype = h->A == 0 ? B200GYM_ACT_I64 : B200GYM_ACT_F32;
    StepArgs s = a;
    void *scratch = nullptr;
    if (summary) {   // one slice of every per-step output, 16-byte aligned pieces
        const size_t obs_bytes = ((size_t)n * D * sizeof(float) + 15) / 16 * 16, act_bytes = (act_row + 15) / 16 * 16;
        const size_t r_bytes = ((size_t)n * sizeof(double) + 15) / 16 * 16, f_bytes = ((size_t)n + 15) / 16 * 16;
        CK(h, cudaMallocAsync(&scratch, obs_bytes + act_bytes + r_bytes + 2 * f_bytes, st));
        unsigned char *base = static_cast<unsigned char *>(scratch);
        s.obs = reinterpret_cast<float *>(base);
        s.actions = base + obs_bytes;
        s.reward = reinterpret_cast<double *>(base + obs_bytes + act_bytes);
        s.terminated = base + obs_bytes + act_bytes + r_bytes;
        s.truncated = s.terminated + f_bytes;
        s.final_obs = nullptr;
    }
    const unsigned blocks = (unsigned)blocks_for(n);
    int rc = 0;
    for (int32_t t = 0; t < T && !rc; t++) {
        const float *obs_in = input(t == 0 ? first_obs : s.obs);
        if (!obs_in) {
            rc = 1;
            break;
        }
        if (!summary) {
            s.actions = static_cast<const unsigned char *>(a.actions) + (size_t)t * act_row;
            s.obs = a.obs + t * n * D;
            s.reward = a.reward + t * n;
            s.terminated = a.terminated + t * n;
            s.truncated = a.truncated + t * n;
            s.final_obs = a.final_obs ? a.final_obs + t * n * D : nullptr;
        }
        if ((rc = hook(t, obs_in, s, false))) break;
        policy<<<blocks, kThreads, smem, st>>>(obs_in, const_cast<void *>(s.actions), args_at(t), s.reward,
                                               s.terminated, s.truncated, n, summary ? t - 1 : -1, 1,
                                               summary && t == 0);
        if (cudaGetLastError() != cudaSuccess) rc = fail(h, "%s: launch failed", kernel);
        else rc = launch_step_box2d(h, s, action_dtype, st);
        if (!rc) rc = hook(t, obs_in, s, true);
    }
    if (!rc && summary) {
        policy<<<blocks, kThreads, smem, st>>>(s.obs, nullptr, args_at(T - 1), s.reward, s.terminated, s.truncated,
                                               n, T - 1, 0, 0);
        if (cudaGetLastError() != cudaSuccess) rc = fail(h, "%s: launch failed", kernel);
    }
    if (!rc && cudaMemcpyAsync(last_obs, s.obs, (size_t)n * D * sizeof(float), cudaMemcpyDeviceToDevice, st))
        rc = fail(h, "%s: copy of the last observations failed", entry);
    if (scratch) cudaFreeAsync(scratch, st);
    return rc;
}

static int launch_rollout_linear_box2d(b200gym *h, const StepArgs &a, int32_t T, float *last_obs,
                                       const float *first_obs, const LinearPolicyArgs &p, bool summary,
                                       cudaStream_t st) {
    void (*policy)(const float *, void *, const LinearPolicyArgs, const double *, const uint8_t *, const uint8_t *,
                   int64_t, int32_t, int, int);
    switch (h->cfg.kind) {
    case B200GYM_LUNARLANDER: policy = linear_policy_kernel<4, 8, true>; break;
    case B200GYM_LUNARLANDER_CONT: policy = linear_policy_kernel<2, 8, false>; break;
    default: policy = linear_policy_kernel<4, 24, false>; break;   // BipedalWalker(Hardcore)
    }
    return launch_rollout_policy_box2d(h, a, T, last_obs, first_obs, [&](int32_t) { return p; }, policy, 0, summary,
                                       st, "linear_policy_kernel", "b200gym_rollout_linear");
}

extern "C" int b200gym_rollout_linear(b200gym_t *h, const float *weight_dev, const float *bias_dev, int per_env,
                                      int32_t T, void *actions_out_dev, float *obs_dev, double *reward_dev,
                                      uint8_t *terminated_dev, uint8_t *truncated_dev, float *final_obs_dev,
                                      double *returns_dev, int32_t *lengths_dev, uint8_t *ended_dev,
                                      float *last_obs_dev, const float *first_obs_dev, void *stream) {
    if (!h) return fail(h, "b200gym_rollout_linear: null handle");
    if (T < 1) return fail(h, "b200gym_rollout_linear: T must be at least 1 (got %d)", T);
    if (!weight_dev || !bias_dev || !last_obs_dev) return fail(h, "b200gym_rollout_linear: null buffer");
    const bool summary = returns_dev != nullptr;
    if (summary ? (!lengths_dev || !ended_dev || actions_out_dev || obs_dev || reward_dev || terminated_dev ||
                   truncated_dev || final_obs_dev)
                : (!actions_out_dev || !obs_dev || !reward_dev || !terminated_dev || !truncated_dev || lengths_dev ||
                   ended_dev))
        return fail(h, "b200gym_rollout_linear: give either the per-step outputs or returns, lengths and ended");
    const bool box2d = h->is_lunar || h->is_walker;
    if (box2d && !first_obs_dev) return fail(h, "b200gym_rollout_linear: a Box2D env needs first_obs_dev");
    const int64_t K = h->A == 0 ? h->NACT : h->A;
    LinearPolicyArgs p{weight_dev, bias_dev, per_env ? K * h->D : 0, per_env ? K : 0, returns_dev, lengths_dev,
                       ended_dev};
    DeviceGuard guard(h->device);
    const StepArgs a = make_args(h, actions_out_dev, obs_dev, reward_dev, terminated_dev, truncated_dev, final_obs_dev);
    cudaStream_t st = (cudaStream_t)stream;
    switch (h->cfg.kind) {
    case B200GYM_CARTPOLE: return launch_rollout_linear_kind<B200GYM_CARTPOLE>(h, a, T, last_obs_dev, p, summary, st);
    case B200GYM_MOUNTAINCAR:
        return launch_rollout_linear_kind<B200GYM_MOUNTAINCAR>(h, a, T, last_obs_dev, p, summary, st);
    case B200GYM_MOUNTAINCAR_CONT:
        return launch_rollout_linear_kind<B200GYM_MOUNTAINCAR_CONT>(h, a, T, last_obs_dev, p, summary, st);
    case B200GYM_PENDULUM: return launch_rollout_linear_kind<B200GYM_PENDULUM>(h, a, T, last_obs_dev, p, summary, st);
    case B200GYM_ACROBOT: return launch_rollout_linear_kind<B200GYM_ACROBOT>(h, a, T, last_obs_dev, p, summary, st);
    case B200GYM_LUNARLANDER:
    case B200GYM_LUNARLANDER_CONT:
    case B200GYM_BIPEDALWALKER:
    case B200GYM_BIPEDALWALKER_HARDCORE:
        return launch_rollout_linear_box2d(h, a, T, last_obs_dev, first_obs_dev, p, summary, st);
    }
    return fail(h, "bad kind %d", h->cfg.kind);
}

// ---- closed-loop rollouts of an MLP policy (b200gym_rollout_mlp) ----
template <int KIND, int ACT>
static int launch_rollout_mlp_kind(b200gym *h, const StepArgs &a, int32_t T, float *last_obs, const MlpPolicyArgs &p,
                                   bool per_env, size_t smem, bool summary, cudaStream_t st) {
    const unsigned blocks = blocks_for(h->n);
    if (per_env) {
        if (summary) rollout_mlp_kernel<KIND, true, true, ACT><<<blocks, kThreads, 0, st>>>(a, T, last_obs, p);
        else rollout_mlp_kernel<KIND, false, true, ACT><<<blocks, kThreads, 0, st>>>(a, T, last_obs, p);
    } else {
        if (summary) rollout_mlp_kernel<KIND, true, false, ACT><<<blocks, kThreads, smem, st>>>(a, T, last_obs, p);
        else rollout_mlp_kernel<KIND, false, false, ACT><<<blocks, kThreads, smem, st>>>(a, T, last_obs, p);
    }
    CK(h, cudaGetLastError());
    return 0;
}

template <int K, int D, bool DISCRETE, int ACT>
static int launch_rollout_mlp_box2d(b200gym *h, const StepArgs &a, int32_t T, float *last_obs, const float *first_obs,
                                    const MlpPolicyArgs &p, bool per_env, size_t smem, bool summary, cudaStream_t st) {
    return launch_rollout_policy_box2d(h, a, T, last_obs, first_obs, [&](int32_t) { return p; },
                                       per_env ? mlp_policy_kernel<K, D, DISCRETE, true, ACT>
                                               : mlp_policy_kernel<K, D, DISCRETE, false, ACT>,
                                       per_env ? 0 : smem, summary, st, "mlp_policy_kernel", "b200gym_rollout_mlp");
}

template <int ACT>
static int launch_rollout_mlp(b200gym *h, const StepArgs &a, int32_t T, float *last_obs, const float *first_obs,
                              const MlpPolicyArgs &p, bool pe, size_t smem, bool summary, cudaStream_t st) {
    switch (h->cfg.kind) {
    case B200GYM_CARTPOLE:
        return launch_rollout_mlp_kind<B200GYM_CARTPOLE, ACT>(h, a, T, last_obs, p, pe, smem, summary, st);
    case B200GYM_MOUNTAINCAR:
        return launch_rollout_mlp_kind<B200GYM_MOUNTAINCAR, ACT>(h, a, T, last_obs, p, pe, smem, summary, st);
    case B200GYM_MOUNTAINCAR_CONT:
        return launch_rollout_mlp_kind<B200GYM_MOUNTAINCAR_CONT, ACT>(h, a, T, last_obs, p, pe, smem, summary, st);
    case B200GYM_PENDULUM:
        return launch_rollout_mlp_kind<B200GYM_PENDULUM, ACT>(h, a, T, last_obs, p, pe, smem, summary, st);
    case B200GYM_ACROBOT:
        return launch_rollout_mlp_kind<B200GYM_ACROBOT, ACT>(h, a, T, last_obs, p, pe, smem, summary, st);
    case B200GYM_LUNARLANDER:
        return launch_rollout_mlp_box2d<4, 8, true, ACT>(h, a, T, last_obs, first_obs, p, pe, smem, summary, st);
    case B200GYM_LUNARLANDER_CONT:
        return launch_rollout_mlp_box2d<2, 8, false, ACT>(h, a, T, last_obs, first_obs, p, pe, smem, summary, st);
    case B200GYM_BIPEDALWALKER:
    case B200GYM_BIPEDALWALKER_HARDCORE:
        return launch_rollout_mlp_box2d<4, 24, false, ACT>(h, a, T, last_obs, first_obs, p, pe, smem, summary, st);
    }
    return fail(h, "bad kind %d", h->cfg.kind);
}

extern "C" int b200gym_rollout_mlp(b200gym_t *h, const float *params_dev, int per_env, int n_layers, int h1, int h2,
                                   int32_t T, void *actions_out_dev, float *obs_dev, double *reward_dev,
                                   uint8_t *terminated_dev, uint8_t *truncated_dev, float *final_obs_dev,
                                   double *returns_dev, int32_t *lengths_dev, uint8_t *ended_dev, float *last_obs_dev,
                                   const float *first_obs_dev, void *stream) {
    return b200gym_rollout_mlp_act(h, params_dev, per_env, n_layers, h1, h2, T, actions_out_dev, obs_dev, reward_dev,
                                   terminated_dev, truncated_dev, final_obs_dev, returns_dev, lengths_dev, ended_dev,
                                   last_obs_dev, first_obs_dev, stream, B200GYM_MLP_RELU);
}

extern "C" int b200gym_rollout_mlp_act(b200gym_t *h, const float *params_dev, int per_env, int n_layers, int h1,
                                       int h2, int32_t T, void *actions_out_dev, float *obs_dev, double *reward_dev,
                                       uint8_t *terminated_dev, uint8_t *truncated_dev, float *final_obs_dev,
                                       double *returns_dev, int32_t *lengths_dev, uint8_t *ended_dev,
                                       float *last_obs_dev, const float *first_obs_dev, void *stream, int activation) {
    if (!h) return fail(h, "b200gym_rollout_mlp: null handle");
    if (activation != B200GYM_MLP_RELU && activation != B200GYM_MLP_TANH)
        return fail(h, "b200gym_rollout_mlp_act: activation must be B200GYM_MLP_RELU or B200GYM_MLP_TANH (got %d)",
                    activation);
    if (n_layers != 1 && n_layers != 2)
        return fail(h, "b200gym_rollout_mlp: n_layers must be 1 or 2 (got %d)", n_layers);
    if (h1 < 1 || h1 > kMlpMaxWidth || (n_layers == 2 && (h2 < 1 || h2 > kMlpMaxWidth)))
        return fail(h, "b200gym_rollout_mlp: hidden widths must be 1 .. %d (got %d, %d)", kMlpMaxWidth, h1, h2);
    if (T < 1) return fail(h, "b200gym_rollout_mlp: T must be at least 1 (got %d)", T);
    if (!params_dev || !last_obs_dev) return fail(h, "b200gym_rollout_mlp: null buffer");
    const bool summary = returns_dev != nullptr;
    if (summary ? (!lengths_dev || !ended_dev || actions_out_dev || obs_dev || reward_dev || terminated_dev ||
                   truncated_dev || final_obs_dev)
                : (!actions_out_dev || !obs_dev || !reward_dev || !terminated_dev || !truncated_dev || lengths_dev ||
                   ended_dev))
        return fail(h, "b200gym_rollout_mlp: give either the per-step outputs or returns, lengths and ended");
    const bool box2d = h->is_lunar || h->is_walker;
    if (box2d && !first_obs_dev) return fail(h, "b200gym_rollout_mlp: a Box2D env needs first_obs_dev");
    if (n_layers == 1) h2 = 0;
    const int64_t K = h->A == 0 ? h->NACT : h->A, D = h->D;
    const int64_t P = h2 == 0 ? h1 * D + h1 + K * h1 + K : h1 * D + h1 + (int64_t)h2 * h1 + h2 + K * h2 + K;
    // 16-byte rows of the second layer: h1 % 4 == 0 puts every row of it at a multiple of 4 floats from the policy's
    // start; a per-env policy's start must itself be 16-byte aligned, the shared copy always is
    const bool vec = h1 % 4 == 0 && (!per_env || (P % 4 == 0 && reinterpret_cast<uintptr_t>(params_dev) % 16 == 0));
    const MlpPolicyArgs p{params_dev, per_env ? P : 0, h1, h2, vec ? 1 : 0, returns_dev, lengths_dev, ended_dev};
    const size_t smem = (size_t)(P + 3) / 4 * 16;   // at most 24.1 KB (BipedalWalker at (64, 64)): no opt-in needed
    DeviceGuard guard(h->device);
    const StepArgs a = make_args(h, actions_out_dev, obs_dev, reward_dev, terminated_dev, truncated_dev, final_obs_dev);
    cudaStream_t st = (cudaStream_t)stream;
    const bool pe = per_env != 0;
    if (activation == B200GYM_MLP_TANH)
        return launch_rollout_mlp<B200GYM_MLP_TANH>(h, a, T, last_obs_dev, first_obs_dev, p, pe, smem, summary, st);
    return launch_rollout_mlp<B200GYM_MLP_RELU>(h, a, T, last_obs_dev, first_obs_dev, p, pe, smem, summary, st);
}

// ---- stochastic rollouts of an MLP policy (b200gym_rollout_mlp_noisy) ----
template <int KIND, int ACT>
static int launch_rollout_mlp_noisy_kind(b200gym *h, const StepArgs &a, int32_t T, float *last_obs,
                                         const MlpNoisyArgs &p, bool per_env, size_t smem, cudaStream_t st) {
    const unsigned blocks = blocks_for(h->n);
    if (per_env) rollout_mlp_noisy_kernel<KIND, true, ACT><<<blocks, kThreads, 0, st>>>(a, T, last_obs, p);
    else rollout_mlp_noisy_kernel<KIND, false, ACT><<<blocks, kThreads, smem, st>>>(a, T, last_obs, p);
    CK(h, cudaGetLastError());
    return 0;
}

// The policy launch of step t reads noise slice t and writes outputs slice t
template <int K, int D, bool DISCRETE, int ACT>
static int launch_rollout_mlp_noisy_box2d(b200gym *h, const StepArgs &a, int32_t T, float *last_obs,
                                          const float *first_obs, const MlpNoisyArgs &p, bool per_env, size_t smem,
                                          cudaStream_t st) {
    const int64_t slice = h->n * K;
    return launch_rollout_policy_box2d(h, a, T, last_obs, first_obs,
                                       [&](int32_t t) {
                                           MlpNoisyArgs q = p;
                                           q.noise = p.noise + t * slice;
                                           q.outputs = p.outputs + t * slice;
                                           return q;
                                       },
                                       per_env ? mlp_noisy_policy_kernel<K, D, DISCRETE, true, ACT>
                                               : mlp_noisy_policy_kernel<K, D, DISCRETE, false, ACT>,
                                       per_env ? 0 : smem, false, st, "mlp_noisy_policy_kernel",
                                       "b200gym_rollout_mlp_noisy");
}

template <int ACT>
static int launch_rollout_mlp_noisy(b200gym *h, const StepArgs &a, int32_t T, float *last_obs, const float *first_obs,
                                    const MlpNoisyArgs &p, bool pe, size_t smem, cudaStream_t st) {
    switch (h->cfg.kind) {
    case B200GYM_CARTPOLE:
        return launch_rollout_mlp_noisy_kind<B200GYM_CARTPOLE, ACT>(h, a, T, last_obs, p, pe, smem, st);
    case B200GYM_MOUNTAINCAR:
        return launch_rollout_mlp_noisy_kind<B200GYM_MOUNTAINCAR, ACT>(h, a, T, last_obs, p, pe, smem, st);
    case B200GYM_MOUNTAINCAR_CONT:
        return launch_rollout_mlp_noisy_kind<B200GYM_MOUNTAINCAR_CONT, ACT>(h, a, T, last_obs, p, pe, smem, st);
    case B200GYM_PENDULUM:
        return launch_rollout_mlp_noisy_kind<B200GYM_PENDULUM, ACT>(h, a, T, last_obs, p, pe, smem, st);
    case B200GYM_ACROBOT:
        return launch_rollout_mlp_noisy_kind<B200GYM_ACROBOT, ACT>(h, a, T, last_obs, p, pe, smem, st);
    case B200GYM_LUNARLANDER:
        return launch_rollout_mlp_noisy_box2d<4, 8, true, ACT>(h, a, T, last_obs, first_obs, p, pe, smem, st);
    case B200GYM_LUNARLANDER_CONT:
        return launch_rollout_mlp_noisy_box2d<2, 8, false, ACT>(h, a, T, last_obs, first_obs, p, pe, smem, st);
    case B200GYM_BIPEDALWALKER:
    case B200GYM_BIPEDALWALKER_HARDCORE:
        return launch_rollout_mlp_noisy_box2d<4, 24, false, ACT>(h, a, T, last_obs, first_obs, p, pe, smem, st);
    }
    return fail(h, "bad kind %d", h->cfg.kind);
}

extern "C" int b200gym_rollout_mlp_noisy(b200gym_t *h, const float *params_dev, int per_env, int n_layers, int h1,
                                         int h2, int32_t T, const float *noise_dev, float *outputs_dev,
                                         void *actions_out_dev, float *obs_dev, double *reward_dev,
                                         uint8_t *terminated_dev, uint8_t *truncated_dev, float *final_obs_dev,
                                         float *last_obs_dev, const float *first_obs_dev, void *stream) {
    return b200gym_rollout_mlp_noisy_act(h, params_dev, per_env, n_layers, h1, h2, T, noise_dev, outputs_dev,
                                         actions_out_dev, obs_dev, reward_dev, terminated_dev, truncated_dev,
                                         final_obs_dev, last_obs_dev, first_obs_dev, stream, B200GYM_MLP_RELU);
}

extern "C" int b200gym_rollout_mlp_noisy_act(b200gym_t *h, const float *params_dev, int per_env, int n_layers, int h1,
                                             int h2, int32_t T, const float *noise_dev, float *outputs_dev,
                                             void *actions_out_dev, float *obs_dev, double *reward_dev,
                                             uint8_t *terminated_dev, uint8_t *truncated_dev, float *final_obs_dev,
                                             float *last_obs_dev, const float *first_obs_dev, void *stream,
                                             int activation) {
    if (!h) return fail(h, "b200gym_rollout_mlp_noisy: null handle");
    if (activation != B200GYM_MLP_RELU && activation != B200GYM_MLP_TANH)
        return fail(h,
                    "b200gym_rollout_mlp_noisy_act: activation must be B200GYM_MLP_RELU or B200GYM_MLP_TANH (got %d)",
                    activation);
    if (n_layers != 1 && n_layers != 2)
        return fail(h, "b200gym_rollout_mlp_noisy: n_layers must be 1 or 2 (got %d)", n_layers);
    if (h1 < 1 || h1 > kMlpMaxWidth || (n_layers == 2 && (h2 < 1 || h2 > kMlpMaxWidth)))
        return fail(h, "b200gym_rollout_mlp_noisy: hidden widths must be 1 .. %d (got %d, %d)", kMlpMaxWidth, h1, h2);
    if (T < 1) return fail(h, "b200gym_rollout_mlp_noisy: T must be at least 1 (got %d)", T);
    if (!params_dev || !noise_dev || !outputs_dev || !actions_out_dev || !obs_dev || !reward_dev || !terminated_dev ||
        !truncated_dev || !last_obs_dev)
        return fail(h, "b200gym_rollout_mlp_noisy: null buffer");
    const bool box2d = h->is_lunar || h->is_walker;
    if (box2d && !first_obs_dev) return fail(h, "b200gym_rollout_mlp_noisy: a Box2D env needs first_obs_dev");
    if (n_layers == 1) h2 = 0;
    const int64_t K = h->A == 0 ? h->NACT : h->A, D = h->D;
    const int64_t P = h2 == 0 ? h1 * D + h1 + K * h1 + K : h1 * D + h1 + (int64_t)h2 * h1 + h2 + K * h2 + K;
    // as b200gym_rollout_mlp
    const bool vec = h1 % 4 == 0 && (!per_env || (P % 4 == 0 && reinterpret_cast<uintptr_t>(params_dev) % 16 == 0));
    const MlpNoisyArgs p{{params_dev, per_env ? P : 0, h1, h2, vec ? 1 : 0, nullptr, nullptr, nullptr}, noise_dev,
                         outputs_dev};
    const size_t smem = (size_t)(P + 3) / 4 * 16;
    DeviceGuard guard(h->device);
    const StepArgs a = make_args(h, actions_out_dev, obs_dev, reward_dev, terminated_dev, truncated_dev, final_obs_dev);
    cudaStream_t st = (cudaStream_t)stream;
    const bool pe = per_env != 0;
    if (activation == B200GYM_MLP_TANH)
        return launch_rollout_mlp_noisy<B200GYM_MLP_TANH>(h, a, T, last_obs_dev, first_obs_dev, p, pe, smem, st);
    return launch_rollout_mlp_noisy<B200GYM_MLP_RELU>(h, a, T, last_obs_dev, first_obs_dev, p, pe, smem, st);
}

// ---- squashed-head MLP rollouts (b200gym_rollout_mlp_head, b200gym_rollout_mlp_noisy_head) ----
// noisy: the noisy kernels (p.noise and p.outputs set), else the deterministic ones, summary mode included
template <int KIND, int ACT, int HEAD>
static int launch_rollout_mlp_head_kind(b200gym *h, const StepArgs &a, int32_t T, float *last_obs,
                                        const MlpHeadArgs &p, bool per_env, size_t smem, bool summary, bool noisy,
                                        cudaStream_t st) {
    const unsigned blocks = blocks_for(h->n);
    if (noisy) {
        if (per_env)
            rollout_mlp_noisy_head_kernel<KIND, true, ACT, HEAD><<<blocks, kThreads, 0, st>>>(a, T, last_obs, p);
        else rollout_mlp_noisy_head_kernel<KIND, false, ACT, HEAD><<<blocks, kThreads, smem, st>>>(a, T, last_obs, p);
    } else if (per_env) {
        if (summary)
            rollout_mlp_head_kernel<KIND, true, true, ACT, HEAD><<<blocks, kThreads, 0, st>>>(a, T, last_obs, p);
        else rollout_mlp_head_kernel<KIND, false, true, ACT, HEAD><<<blocks, kThreads, 0, st>>>(a, T, last_obs, p);
    } else {
        if (summary)
            rollout_mlp_head_kernel<KIND, true, false, ACT, HEAD><<<blocks, kThreads, smem, st>>>(a, T, last_obs, p);
        else rollout_mlp_head_kernel<KIND, false, false, ACT, HEAD><<<blocks, kThreads, smem, st>>>(a, T, last_obs, p);
    }
    CK(h, cudaGetLastError());
    return 0;
}

// The policy launch of step t of a noisy rollout reads noise slice t and writes outputs slice t
template <int K, int D, int ACT, int HEAD>
static int launch_rollout_mlp_head_box2d(b200gym *h, const StepArgs &a, int32_t T, float *last_obs,
                                         const float *first_obs, const MlpHeadArgs &p, bool per_env, size_t smem,
                                         bool summary, bool noisy, cudaStream_t st) {
    constexpr int A = HEAD == B200GYM_HEAD_TANH_NORMAL ? K / 2 : K;
    if (noisy) {
        const int64_t n = h->n;
        return launch_rollout_policy_box2d(h, a, T, last_obs, first_obs,
                                           [&](int32_t t) {
                                               MlpHeadArgs q = p;
                                               q.noise = p.noise + t * n * A;
                                               q.outputs = p.outputs + t * n * K;
                                               return q;
                                           },
                                           per_env ? mlp_noisy_head_policy_kernel<K, D, true, ACT, HEAD>
                                                   : mlp_noisy_head_policy_kernel<K, D, false, ACT, HEAD>,
                                           per_env ? 0 : smem, false, st, "mlp_noisy_head_policy_kernel",
                                           "b200gym_rollout_mlp_noisy_head");
    }
    return launch_rollout_policy_box2d(h, a, T, last_obs, first_obs, [&](int32_t) { return p; },
                                       per_env ? mlp_head_policy_kernel<K, D, true, ACT, HEAD>
                                               : mlp_head_policy_kernel<K, D, false, ACT, HEAD>,
                                       per_env ? 0 : smem, summary, st, "mlp_head_policy_kernel",
                                       "b200gym_rollout_mlp_head");
}

template <int ACT, int HEAD>
static int launch_rollout_mlp_head(b200gym *h, const StepArgs &a, int32_t T, float *last_obs, const float *first_obs,
                                   const MlpHeadArgs &p, bool pe, size_t smem, bool summary, bool noisy,
                                   cudaStream_t st) {
    switch (h->cfg.kind) {
    case B200GYM_MOUNTAINCAR_CONT:
        return launch_rollout_mlp_head_kind<B200GYM_MOUNTAINCAR_CONT, ACT, HEAD>(h, a, T, last_obs, p, pe, smem,
                                                                                 summary, noisy, st);
    case B200GYM_PENDULUM:
        return launch_rollout_mlp_head_kind<B200GYM_PENDULUM, ACT, HEAD>(h, a, T, last_obs, p, pe, smem, summary,
                                                                         noisy, st);
    case B200GYM_LUNARLANDER_CONT:
        return launch_rollout_mlp_head_box2d<head_outputs<HEAD>(2), 8, ACT, HEAD>(h, a, T, last_obs, first_obs, p, pe,
                                                                                  smem, summary, noisy, st);
    case B200GYM_BIPEDALWALKER:
    case B200GYM_BIPEDALWALKER_HARDCORE:
        return launch_rollout_mlp_head_box2d<head_outputs<HEAD>(4), 24, ACT, HEAD>(h, a, T, last_obs, first_obs, p,
                                                                                   pe, smem, summary, noisy, st);
    }
    return fail(h, "bad kind %d", h->cfg.kind);
}

// The checks and launches of both entry points: noisy (b200gym_rollout_mlp_noisy_head) reads noise_dev and writes
// outputs_dev, and has no summary mode; `what` names the entry point in the messages
static int rollout_mlp_head(const char *what, b200gym_t *h, const float *params_dev, int per_env, int n_layers, int h1,
                            int h2, int32_t T, bool noisy, const float *noise_dev, float *outputs_dev,
                            void *actions_out_dev, float *obs_dev, double *reward_dev, uint8_t *terminated_dev,
                            uint8_t *truncated_dev, float *final_obs_dev, double *returns_dev, int32_t *lengths_dev,
                            uint8_t *ended_dev, float *last_obs_dev, const float *first_obs_dev, void *stream,
                            int activation, int head) {
    if (!h) return fail(h, "%s: null handle", what);
    if (head != B200GYM_HEAD_TANH && head != B200GYM_HEAD_TANH_NORMAL)
        return fail(h, "%s: head must be B200GYM_HEAD_TANH or B200GYM_HEAD_TANH_NORMAL (got %d)", what, head);
    if (activation != B200GYM_MLP_RELU && activation != B200GYM_MLP_TANH)
        return fail(h, "%s: activation must be B200GYM_MLP_RELU or B200GYM_MLP_TANH (got %d)", what, activation);
    const int kind = h->cfg.kind;
    if (kind != B200GYM_MOUNTAINCAR_CONT && kind != B200GYM_PENDULUM && kind != B200GYM_LUNARLANDER_CONT &&
        kind != B200GYM_BIPEDALWALKER && kind != B200GYM_BIPEDALWALKER_HARDCORE)
        return fail(h, "%s: a head needs a Box action space (kind %d is Discrete)", what, kind);
    if (n_layers != 1 && n_layers != 2) return fail(h, "%s: n_layers must be 1 or 2 (got %d)", what, n_layers);
    if (h1 < 1 || h1 > kMlpMaxWidth || (n_layers == 2 && (h2 < 1 || h2 > kMlpMaxWidth)))
        return fail(h, "%s: hidden widths must be 1 .. %d (got %d, %d)", what, kMlpMaxWidth, h1, h2);
    if (T < 1) return fail(h, "%s: T must be at least 1 (got %d)", what, T);
    if (!params_dev || !last_obs_dev || (noisy && (!noise_dev || !outputs_dev)))
        return fail(h, "%s: null buffer", what);
    const bool summary = returns_dev != nullptr;
    if (summary ? (noisy || !lengths_dev || !ended_dev || actions_out_dev || obs_dev || reward_dev || terminated_dev ||
                   truncated_dev || final_obs_dev)
                : (!actions_out_dev || !obs_dev || !reward_dev || !terminated_dev || !truncated_dev || lengths_dev ||
                   ended_dev))
        return fail(h, "%s: give %s", what,
                    noisy ? "the per-step outputs" : "either the per-step outputs or returns, lengths and ended");
    if ((h->is_lunar || h->is_walker) && !first_obs_dev) return fail(h, "%s: a Box2D env needs first_obs_dev", what);
    if (n_layers == 1) h2 = 0;
    const int64_t K = head == B200GYM_HEAD_TANH_NORMAL ? 2 * h->A : h->A, D = h->D;
    const int64_t P = h2 == 0 ? h1 * D + h1 + K * h1 + K : h1 * D + h1 + (int64_t)h2 * h1 + h2 + K * h2 + K;
    // as b200gym_rollout_mlp
    const bool vec = h1 % 4 == 0 && (!per_env || (P % 4 == 0 && reinterpret_cast<uintptr_t>(params_dev) % 16 == 0));
    // the kind's action bounds, and CleanRL's action_scale and action_bias from them, in float32
    const float high = kind == B200GYM_PENDULUM ? 2.0f : 1.0f, low = -high;
    const HeadBounds bounds{low, high, (high - low) / 2.0f, (high + low) / 2.0f};
    const MlpHeadArgs p{{params_dev, per_env ? P : 0, h1, h2, vec ? 1 : 0, returns_dev, lengths_dev, ended_dev},
                        noise_dev, outputs_dev, bounds};
    const size_t smem = (size_t)(P + 3) / 4 * 16;   // at most 24.5 KB (BipedalWalker's SAC actor at (64, 64))
    DeviceGuard guard(h->device);
    const StepArgs a = make_args(h, actions_out_dev, obs_dev, reward_dev, terminated_dev, truncated_dev, final_obs_dev);
    cudaStream_t st = (cudaStream_t)stream;
    const bool pe = per_env != 0;
    if (activation == B200GYM_MLP_TANH) {
        if (head == B200GYM_HEAD_TANH_NORMAL)
            return launch_rollout_mlp_head<B200GYM_MLP_TANH, B200GYM_HEAD_TANH_NORMAL>(
                h, a, T, last_obs_dev, first_obs_dev, p, pe, smem, summary, noisy, st);
        return launch_rollout_mlp_head<B200GYM_MLP_TANH, B200GYM_HEAD_TANH>(h, a, T, last_obs_dev, first_obs_dev, p, pe,
                                                                            smem, summary, noisy, st);
    }
    if (head == B200GYM_HEAD_TANH_NORMAL)
        return launch_rollout_mlp_head<B200GYM_MLP_RELU, B200GYM_HEAD_TANH_NORMAL>(h, a, T, last_obs_dev, first_obs_dev,
                                                                                   p, pe, smem, summary, noisy, st);
    return launch_rollout_mlp_head<B200GYM_MLP_RELU, B200GYM_HEAD_TANH>(h, a, T, last_obs_dev, first_obs_dev, p, pe,
                                                                        smem, summary, noisy, st);
}

extern "C" int b200gym_rollout_mlp_head(b200gym_t *h, const float *params_dev, int per_env, int n_layers, int h1,
                                        int h2, int32_t T, void *actions_out_dev, float *obs_dev, double *reward_dev,
                                        uint8_t *terminated_dev, uint8_t *truncated_dev, float *final_obs_dev,
                                        double *returns_dev, int32_t *lengths_dev, uint8_t *ended_dev,
                                        float *last_obs_dev, const float *first_obs_dev, void *stream, int activation,
                                        int head) {
    return rollout_mlp_head("b200gym_rollout_mlp_head", h, params_dev, per_env, n_layers, h1, h2, T, false, nullptr,
                            nullptr, actions_out_dev, obs_dev, reward_dev, terminated_dev, truncated_dev,
                            final_obs_dev, returns_dev, lengths_dev, ended_dev, last_obs_dev, first_obs_dev, stream,
                            activation, head);
}

extern "C" int b200gym_rollout_mlp_noisy_head(b200gym_t *h, const float *params_dev, int per_env, int n_layers, int h1,
                                              int h2, int32_t T, const float *noise_dev, float *outputs_dev,
                                              void *actions_out_dev, float *obs_dev, double *reward_dev,
                                              uint8_t *terminated_dev, uint8_t *truncated_dev, float *final_obs_dev,
                                              float *last_obs_dev, const float *first_obs_dev, void *stream,
                                              int activation, int head) {
    return rollout_mlp_head("b200gym_rollout_mlp_noisy_head", h, params_dev, per_env, n_layers, h1, h2, T, true,
                            noise_dev, outputs_dev, actions_out_dev, obs_dev, reward_dev, terminated_dev,
                            truncated_dev, final_obs_dev, nullptr, nullptr, nullptr, last_obs_dev, first_obs_dev,
                            stream, activation, head);
}

// ---- on-policy collection with a critic (b200gym_rollout_actor_critic) ----
static int launch_gae(b200gym *h, const StepArgs &a, int32_t T, const ActorCriticArgs &p, float g, float gl,
                      cudaStream_t st) {
    gae_kernel<<<blocks_for(h->n), kThreads, 0, st>>>(a.reward, a.terminated, a.truncated, p.values, p.advantages, h->n,
                                                      T, g, gl);
    CK(h, cudaGetLastError());
    return 0;
}

template <int KIND, int ACT>
static int launch_rollout_actor_critic_kind(b200gym *h, const StepArgs &a, int32_t T, float *last_obs,
                                            const ActorCriticArgs &p, size_t smem, float g, float gl,
                                            cudaStream_t st) {
    rollout_actor_critic_kernel<KIND, ACT><<<blocks_for(h->n), kThreads, smem, st>>>(a, T, last_obs, p);
    CK(h, cudaGetLastError());
    return launch_gae(h, a, T, p, g, gl, st);
}

// Composed launch by launch: around the noisy policy launch and step sequence of step t, the critic (mlp_policy_kernel
// with K = 1, whose Box "action" is V) on the step's input rows into values[t], and after it on the step's final
// observation rows into advantages[t], the holding slot gae_kernel reads where the step truncated without terminating
// (every row is evaluated, the others are overwritten unread).  Then the critic on the last observations into
// values[T], and gae_kernel
template <int K, int D, bool DISCRETE, int ACT>
static int launch_rollout_actor_critic_box2d(b200gym *h, const StepArgs &a, int32_t T, float *last_obs,
                                             const float *first_obs, const ActorCriticArgs &p, size_t smem_actor,
                                             size_t smem_critic, float g, float gl, cudaStream_t st) {
    const int64_t n = h->n, slice = n * K;
    const MlpPolicyArgs c{p.critic, 0, p.actor.mlp.h1, p.actor.mlp.h2, p.actor.mlp.vec, nullptr, nullptr, nullptr};
    const unsigned blocks = blocks_for(n);
    auto critic = [&](const float *obs, float *out) {
        mlp_policy_kernel<1, D, false, false, ACT><<<blocks, kThreads, smem_critic, st>>>(obs, out, c, nullptr, nullptr,
                                                                                        nullptr, n, -1, 1, 0);
        return cudaGetLastError() != cudaSuccess ? fail(h, "mlp_policy_kernel (critic): launch failed") : 0;
    };
    int rc = launch_rollout_policy_box2d(
        h, a, T, last_obs, first_obs,
        [&](int32_t t) {
            MlpNoisyArgs q = p.actor;
            q.noise = p.actor.noise + t * slice;
            q.outputs = p.actor.outputs + t * slice;
            return q;
        },
        mlp_noisy_policy_kernel<K, D, DISCRETE, false, ACT>, smem_actor, false, st, "mlp_noisy_policy_kernel",
        "b200gym_rollout_actor_critic", [&](int32_t t, const float *obs_in, const StepArgs &s, bool after) {
            return after ? critic(s.final_obs, p.advantages + t * n) : critic(obs_in, p.values + t * n);
        });
    if (!rc) rc = critic(last_obs, p.values + (int64_t)T * n);
    return rc ? rc : launch_gae(h, a, T, p, g, gl, st);
}

template <int ACT>
static int launch_rollout_actor_critic(b200gym *h, const StepArgs &a, int32_t T, float *last_obs,
                                       const float *first_obs, const ActorCriticArgs &p, size_t smem_actor,
                                       size_t smem_critic, float g, float gl, cudaStream_t st) {
    const size_t smem = smem_actor + smem_critic;
    switch (h->cfg.kind) {
    case B200GYM_CARTPOLE:
        return launch_rollout_actor_critic_kind<B200GYM_CARTPOLE, ACT>(h, a, T, last_obs, p, smem, g, gl, st);
    case B200GYM_MOUNTAINCAR:
        return launch_rollout_actor_critic_kind<B200GYM_MOUNTAINCAR, ACT>(h, a, T, last_obs, p, smem, g, gl, st);
    case B200GYM_MOUNTAINCAR_CONT:
        return launch_rollout_actor_critic_kind<B200GYM_MOUNTAINCAR_CONT, ACT>(h, a, T, last_obs, p, smem, g, gl, st);
    case B200GYM_PENDULUM:
        return launch_rollout_actor_critic_kind<B200GYM_PENDULUM, ACT>(h, a, T, last_obs, p, smem, g, gl, st);
    case B200GYM_ACROBOT:
        return launch_rollout_actor_critic_kind<B200GYM_ACROBOT, ACT>(h, a, T, last_obs, p, smem, g, gl, st);
    case B200GYM_LUNARLANDER:
        return launch_rollout_actor_critic_box2d<4, 8, true, ACT>(h, a, T, last_obs, first_obs, p, smem_actor,
                                                                  smem_critic, g, gl, st);
    case B200GYM_LUNARLANDER_CONT:
        return launch_rollout_actor_critic_box2d<2, 8, false, ACT>(h, a, T, last_obs, first_obs, p, smem_actor,
                                                                   smem_critic, g, gl, st);
    case B200GYM_BIPEDALWALKER:
    case B200GYM_BIPEDALWALKER_HARDCORE:
        return launch_rollout_actor_critic_box2d<4, 24, false, ACT>(h, a, T, last_obs, first_obs, p, smem_actor,
                                                                    smem_critic, g, gl, st);
    }
    return fail(h, "bad kind %d", h->cfg.kind);
}

extern "C" int b200gym_rollout_actor_critic(b200gym_t *h, const float *actor_dev, const float *critic_dev,
                                            int n_layers, int h1, int h2, int32_t T, const float *noise_dev,
                                            float *outputs_dev, void *actions_out_dev, float *obs_dev,
                                            double *reward_dev, uint8_t *terminated_dev, uint8_t *truncated_dev,
                                            float *final_obs_dev, float *values_dev, float *advantages_dev,
                                            float gamma, float gamma_lambda, float *last_obs_dev,
                                            const float *first_obs_dev, void *stream, int activation) {
    if (!h) return fail(h, "b200gym_rollout_actor_critic: null handle");
    if (activation != B200GYM_MLP_RELU && activation != B200GYM_MLP_TANH)
        return fail(h, "b200gym_rollout_actor_critic: activation must be B200GYM_MLP_RELU or B200GYM_MLP_TANH (got %d)",
                    activation);
    if (n_layers != 1 && n_layers != 2)
        return fail(h, "b200gym_rollout_actor_critic: n_layers must be 1 or 2 (got %d)", n_layers);
    if (h1 < 1 || h1 > kMlpMaxWidth || (n_layers == 2 && (h2 < 1 || h2 > kMlpMaxWidth)))
        return fail(h, "b200gym_rollout_actor_critic: hidden widths must be 1 .. %d (got %d, %d)", kMlpMaxWidth, h1,
                    h2);
    if (T < 1) return fail(h, "b200gym_rollout_actor_critic: T must be at least 1 (got %d)", T);
    if (!(gamma >= 0.0f && gamma <= 1.0f && gamma_lambda >= 0.0f && gamma_lambda <= 1.0f))
        return fail(h, "b200gym_rollout_actor_critic: gamma and gamma_lambda must be in [0, 1] (got %g, %g)",
                    (double)gamma, (double)gamma_lambda);
    if (!actor_dev || !critic_dev || !noise_dev || !outputs_dev || !actions_out_dev || !obs_dev || !reward_dev ||
        !terminated_dev || !truncated_dev || !values_dev || !advantages_dev || !last_obs_dev)
        return fail(h, "b200gym_rollout_actor_critic: null buffer");
    if (!final_obs_dev || !h->cfg.autoreset)
        return fail(h, "b200gym_rollout_actor_critic: the truncation bootstrap needs autoreset and final_obs_dev");
    const bool box2d = h->is_lunar || h->is_walker;
    if (box2d && !first_obs_dev) return fail(h, "b200gym_rollout_actor_critic: a Box2D env needs first_obs_dev");
    if (n_layers == 1) h2 = 0;
    const int64_t K = h->A == 0 ? h->NACT : h->A, D = h->D;
    const int64_t Pa = h2 == 0 ? h1 * D + h1 + K * h1 + K : h1 * D + h1 + (int64_t)h2 * h1 + h2 + K * h2 + K;
    const int64_t Pc = h2 == 0 ? h1 * D + h1 + h1 + 1 : h1 * D + h1 + (int64_t)h2 * h1 + h2 + h2 + 1;
    // the shared copies start 16-byte aligned, so h1 % 4 == 0 is all the 16-byte rows of either net need
    const bool vec = h1 % 4 == 0;
    const ActorCriticArgs p{{{actor_dev, 0, h1, h2, vec ? 1 : 0, nullptr, nullptr, nullptr}, noise_dev, outputs_dev},
                            critic_dev, values_dev, advantages_dev};
    // at most 37.9 KB (Acrobot at (64, 64): 4803 + 4673 floats): no opt-in needed
    const size_t smem_actor = (size_t)(Pa + 3) / 4 * 16, smem_critic = (size_t)(Pc + 3) / 4 * 16;
    DeviceGuard guard(h->device);
    const StepArgs a = make_args(h, actions_out_dev, obs_dev, reward_dev, terminated_dev, truncated_dev, final_obs_dev);
    cudaStream_t st = (cudaStream_t)stream;
    if (activation == B200GYM_MLP_TANH)
        return launch_rollout_actor_critic<B200GYM_MLP_TANH>(h, a, T, last_obs_dev, first_obs_dev, p, smem_actor,
                                                             smem_critic, gamma, gamma_lambda, st);
    return launch_rollout_actor_critic<B200GYM_MLP_RELU>(h, a, T, last_obs_dev, first_obs_dev, p, smem_actor,
                                                         smem_critic, gamma, gamma_lambda, st);
}

// ---- normalised observations and rewards (b200gym_rollout_mlp_noisy_norm, b200gym_rollout_actor_critic_norm) ----
// The Box2D kinds' network inputs: norm_rows_kernel from the observation rows o into the handle's scratch rows, made
// on first use (these kinds refuse CUDA-graph capture).  nullptr on failure, with the error set
static const float *launch_norm_rows(b200gym *h, const float *o, const ObsNormArgs &q, cudaStream_t st,
                                     const char *entry) {
    const int64_t total = h->n * h->D;
    if (!h->norm_rows && cudaMalloc((void **)&h->norm_rows, (size_t)total * sizeof(float)) != cudaSuccess) {
        h->norm_rows = nullptr;
        fail(h, "%s: cannot allocate the normalised input rows", entry);
        return nullptr;
    }
    norm_rows_kernel<<<blocks_for(total), kThreads, 0, st>>>(o, h->norm_rows, total, (int)h->D, q);
    if (cudaGetLastError() != cudaSuccess) {
        fail(h, "norm_rows_kernel: launch failed");
        return nullptr;
    }
    return h->norm_rows;
}

// The statistics checks both entry points share; `what` names the caller in the error
static int norm_args_check(b200gym *h, const char *what, const double *mean, const double *var, double eps, float clip) {
    if ((mean == nullptr) != (var == nullptr)) return fail(h, "%s: give both obs_mean_dev and obs_var_dev, or neither", what);
    if (!(eps >= 0.0 && std::isfinite(eps))) return fail(h, "%s: eps must be finite and at least 0 (got %g)", what, eps);
    if (!(clip > 0.0f)) return fail(h, "%s: clip_obs must be above 0, +inf for none (got %g)", what, (double)clip);
    if (!mean && !std::isinf(clip)) return fail(h, "%s: clip_obs needs obs_mean_dev and obs_var_dev", what);
    if (mean && h->D > kMaxNormDim) return fail(h, "%s: obs_dim %d is above %d", what, h->D, kMaxNormDim);
    return 0;
}

template <int KIND, int ACT>
static int launch_rollout_mlp_noisy_norm_kind(b200gym *h, const StepArgs &a, int32_t T, float *last_obs,
                                              const MlpNoisyArgs &p, const ObsNormArgs &q, size_t smem,
                                              cudaStream_t st) {
    rollout_mlp_noisy_norm_kernel<KIND, ACT><<<blocks_for(h->n), kThreads, smem, st>>>(a, T, last_obs, p, q);
    CK(h, cudaGetLastError());
    return 0;
}

// launch_rollout_mlp_noisy_box2d's sequence with the policy reading the normalised rows of its input
template <int K, int D, bool DISCRETE, int ACT>
static int launch_rollout_mlp_noisy_norm_box2d(b200gym *h, const StepArgs &a, int32_t T, float *last_obs,
                                               const float *first_obs, const MlpNoisyArgs &p, const ObsNormArgs &q,
                                               size_t smem, cudaStream_t st) {
    const int64_t slice = h->n * K;
    const char *entry = "b200gym_rollout_mlp_noisy_norm";
    return launch_rollout_policy_box2d(
        h, a, T, last_obs, first_obs,
        [&](int32_t t) {
            MlpNoisyArgs r = p;
            r.noise = p.noise + t * slice;
            r.outputs = p.outputs + t * slice;
            return r;
        },
        mlp_noisy_policy_kernel<K, D, DISCRETE, false, ACT>, smem, false, st, "mlp_noisy_policy_kernel", entry,
        NoStepHook{}, [&](const float *o) { return launch_norm_rows(h, o, q, st, entry); });
}

template <int ACT>
static int launch_rollout_mlp_noisy_norm(b200gym *h, const StepArgs &a, int32_t T, float *last_obs,
                                         const float *first_obs, const MlpNoisyArgs &p, const ObsNormArgs &q,
                                         size_t smem, cudaStream_t st) {
    switch (h->cfg.kind) {
    case B200GYM_CARTPOLE:
        return launch_rollout_mlp_noisy_norm_kind<B200GYM_CARTPOLE, ACT>(h, a, T, last_obs, p, q, smem, st);
    case B200GYM_MOUNTAINCAR:
        return launch_rollout_mlp_noisy_norm_kind<B200GYM_MOUNTAINCAR, ACT>(h, a, T, last_obs, p, q, smem, st);
    case B200GYM_MOUNTAINCAR_CONT:
        return launch_rollout_mlp_noisy_norm_kind<B200GYM_MOUNTAINCAR_CONT, ACT>(h, a, T, last_obs, p, q, smem, st);
    case B200GYM_PENDULUM:
        return launch_rollout_mlp_noisy_norm_kind<B200GYM_PENDULUM, ACT>(h, a, T, last_obs, p, q, smem, st);
    case B200GYM_ACROBOT:
        return launch_rollout_mlp_noisy_norm_kind<B200GYM_ACROBOT, ACT>(h, a, T, last_obs, p, q, smem, st);
    case B200GYM_LUNARLANDER:
        return launch_rollout_mlp_noisy_norm_box2d<4, 8, true, ACT>(h, a, T, last_obs, first_obs, p, q, smem, st);
    case B200GYM_LUNARLANDER_CONT:
        return launch_rollout_mlp_noisy_norm_box2d<2, 8, false, ACT>(h, a, T, last_obs, first_obs, p, q, smem, st);
    case B200GYM_BIPEDALWALKER:
    case B200GYM_BIPEDALWALKER_HARDCORE:
        return launch_rollout_mlp_noisy_norm_box2d<4, 24, false, ACT>(h, a, T, last_obs, first_obs, p, q, smem, st);
    }
    return fail(h, "bad kind %d", h->cfg.kind);
}

extern "C" int b200gym_rollout_mlp_noisy_norm(b200gym_t *h, const float *params_dev, int per_env, int n_layers, int h1,
                                              int h2, int32_t T, const float *noise_dev, float *outputs_dev,
                                              void *actions_out_dev, float *obs_dev, double *reward_dev,
                                              uint8_t *terminated_dev, uint8_t *truncated_dev, float *final_obs_dev,
                                              float *last_obs_dev, const float *first_obs_dev, void *stream,
                                              int activation, const double *obs_mean_dev, const double *obs_var_dev,
                                              double eps, float clip_obs) {
    const char *what = "b200gym_rollout_mlp_noisy_norm";
    if (!h) return fail(h, "%s: null handle", what);
    if (int rc = norm_args_check(h, what, obs_mean_dev, obs_var_dev, eps, clip_obs)) return rc;
    if (!obs_mean_dev)   // not normalised: b200gym_rollout_mlp_noisy_act's own checks and kernels
        return b200gym_rollout_mlp_noisy_act(h, params_dev, per_env, n_layers, h1, h2, T, noise_dev, outputs_dev,
                                             actions_out_dev, obs_dev, reward_dev, terminated_dev, truncated_dev,
                                             final_obs_dev, last_obs_dev, first_obs_dev, stream, activation);
    if (activation != B200GYM_MLP_RELU && activation != B200GYM_MLP_TANH)
        return fail(h, "%s: activation must be B200GYM_MLP_RELU or B200GYM_MLP_TANH (got %d)", what, activation);
    if (per_env) return fail(h, "%s: normalised inputs need one policy shared by every env (per_env = 0)", what);
    if (n_layers != 1 && n_layers != 2) return fail(h, "%s: n_layers must be 1 or 2 (got %d)", what, n_layers);
    if (h1 < 1 || h1 > kMlpMaxWidth || (n_layers == 2 && (h2 < 1 || h2 > kMlpMaxWidth)))
        return fail(h, "%s: hidden widths must be 1 .. %d (got %d, %d)", what, kMlpMaxWidth, h1, h2);
    if (T < 1) return fail(h, "%s: T must be at least 1 (got %d)", what, T);
    if (!params_dev || !noise_dev || !outputs_dev || !actions_out_dev || !obs_dev || !reward_dev || !terminated_dev ||
        !truncated_dev || !last_obs_dev)
        return fail(h, "%s: null buffer", what);
    const bool box2d = h->is_lunar || h->is_walker;
    if (box2d && !first_obs_dev) return fail(h, "%s: a Box2D env needs first_obs_dev", what);
    if (n_layers == 1) h2 = 0;
    const int64_t K = h->A == 0 ? h->NACT : h->A, D = h->D;
    const int64_t P = h2 == 0 ? h1 * D + h1 + K * h1 + K : h1 * D + h1 + (int64_t)h2 * h1 + h2 + K * h2 + K;
    const bool vec = h1 % 4 == 0;   // the shared copy starts 16-byte aligned
    const MlpNoisyArgs p{{params_dev, 0, h1, h2, vec ? 1 : 0, nullptr, nullptr, nullptr}, noise_dev, outputs_dev};
    const ObsNormArgs q{obs_mean_dev, obs_var_dev, eps, clip_obs};
    const size_t smem = (size_t)(P + 3) / 4 * 16;
    DeviceGuard guard(h->device);
    const StepArgs a = make_args(h, actions_out_dev, obs_dev, reward_dev, terminated_dev, truncated_dev, final_obs_dev);
    cudaStream_t st = (cudaStream_t)stream;
    if (activation == B200GYM_MLP_TANH)
        return launch_rollout_mlp_noisy_norm<B200GYM_MLP_TANH>(h, a, T, last_obs_dev, first_obs_dev, p, q, smem, st);
    return launch_rollout_mlp_noisy_norm<B200GYM_MLP_RELU>(h, a, T, last_obs_dev, first_obs_dev, p, q, smem, st);
}

// launch_gae, or gae_scaled_kernel where the rewards are scaled (ret_var not null)
static int launch_gae_norm(b200gym *h, const StepArgs &a, int32_t T, const ActorCriticArgs &p, float g, float gl,
                           const double *ret_var, double eps, float clip_r, cudaStream_t st) {
    if (!ret_var) return launch_gae(h, a, T, p, g, gl, st);
    gae_scaled_kernel<<<blocks_for(h->n), kThreads, 0, st>>>(a.reward, a.terminated, a.truncated, p.values,
                                                             p.advantages, h->n, T, g, gl, ret_var, eps, clip_r);
    CK(h, cudaGetLastError());
    return 0;
}

// The rollout launch: rollout_actor_critic_norm_kernel, or rollout_actor_critic_kernel where the observations are not
// normalised (q.mean null: only the rewards are)
template <int KIND, int ACT>
static int launch_rollout_actor_critic_norm_kind(b200gym *h, const StepArgs &a, int32_t T, float *last_obs,
                                                 const ActorCriticArgs &p, const ObsNormArgs &q, size_t smem,
                                                 cudaStream_t st) {
    if (q.mean) rollout_actor_critic_norm_kernel<KIND, ACT><<<blocks_for(h->n), kThreads, smem, st>>>(a, T, last_obs, p, q);
    else rollout_actor_critic_kernel<KIND, ACT><<<blocks_for(h->n), kThreads, smem, st>>>(a, T, last_obs, p);
    CK(h, cudaGetLastError());
    return 0;
}

// launch_rollout_actor_critic_box2d's sequence with the critic and the policy reading the normalised rows of their
// input (a norm_rows_kernel launch before them), and each critic launch on final or last observations after one too
template <int K, int D, bool DISCRETE, int ACT>
static int launch_rollout_actor_critic_norm_box2d(b200gym *h, const StepArgs &a, int32_t T, float *last_obs,
                                                  const float *first_obs, const ActorCriticArgs &p,
                                                  const ObsNormArgs &q, size_t smem_actor, size_t smem_critic,
                                                  cudaStream_t st) {
    const int64_t n = h->n, slice = n * K;
    const char *entry = "b200gym_rollout_actor_critic_norm";
    const MlpPolicyArgs c{p.critic, 0, p.actor.mlp.h1, p.actor.mlp.h2, p.actor.mlp.vec, nullptr, nullptr, nullptr};
    const unsigned blocks = blocks_for(n);
    auto input = [&](const float *o) { return q.mean ? launch_norm_rows(h, o, q, st, entry) : o; };
    auto critic = [&](const float *obs, float *out) {
        if (!obs) return 1;
        mlp_policy_kernel<1, D, false, false, ACT><<<blocks, kThreads, smem_critic, st>>>(obs, out, c, nullptr, nullptr,
                                                                                        nullptr, n, -1, 1, 0);
        return cudaGetLastError() != cudaSuccess ? fail(h, "mlp_policy_kernel (critic): launch failed") : 0;
    };
    int rc = launch_rollout_policy_box2d(
        h, a, T, last_obs, first_obs,
        [&](int32_t t) {
            MlpNoisyArgs r = p.actor;
            r.noise = p.actor.noise + t * slice;
            r.outputs = p.actor.outputs + t * slice;
            return r;
        },
        mlp_noisy_policy_kernel<K, D, DISCRETE, false, ACT>, smem_actor, false, st, "mlp_noisy_policy_kernel", entry,
        [&](int32_t t, const float *obs_in, const StepArgs &s, bool after) {
            return after ? critic(input(s.final_obs), p.advantages + t * n) : critic(obs_in, p.values + t * n);
        },
        input);
    if (!rc) rc = critic(input(last_obs), p.values + (int64_t)T * n);
    return rc;
}

template <int ACT>
static int launch_rollout_actor_critic_norm(b200gym *h, const StepArgs &a, int32_t T, float *last_obs,
                                            const float *first_obs, const ActorCriticArgs &p, const ObsNormArgs &q,
                                            size_t smem_actor, size_t smem_critic, cudaStream_t st) {
    const size_t smem = smem_actor + smem_critic;
    switch (h->cfg.kind) {
    case B200GYM_CARTPOLE:
        return launch_rollout_actor_critic_norm_kind<B200GYM_CARTPOLE, ACT>(h, a, T, last_obs, p, q, smem, st);
    case B200GYM_MOUNTAINCAR:
        return launch_rollout_actor_critic_norm_kind<B200GYM_MOUNTAINCAR, ACT>(h, a, T, last_obs, p, q, smem, st);
    case B200GYM_MOUNTAINCAR_CONT:
        return launch_rollout_actor_critic_norm_kind<B200GYM_MOUNTAINCAR_CONT, ACT>(h, a, T, last_obs, p, q, smem, st);
    case B200GYM_PENDULUM:
        return launch_rollout_actor_critic_norm_kind<B200GYM_PENDULUM, ACT>(h, a, T, last_obs, p, q, smem, st);
    case B200GYM_ACROBOT:
        return launch_rollout_actor_critic_norm_kind<B200GYM_ACROBOT, ACT>(h, a, T, last_obs, p, q, smem, st);
    case B200GYM_LUNARLANDER:
        return launch_rollout_actor_critic_norm_box2d<4, 8, true, ACT>(h, a, T, last_obs, first_obs, p, q, smem_actor,
                                                                       smem_critic, st);
    case B200GYM_LUNARLANDER_CONT:
        return launch_rollout_actor_critic_norm_box2d<2, 8, false, ACT>(h, a, T, last_obs, first_obs, p, q, smem_actor,
                                                                        smem_critic, st);
    case B200GYM_BIPEDALWALKER:
    case B200GYM_BIPEDALWALKER_HARDCORE:
        return launch_rollout_actor_critic_norm_box2d<4, 24, false, ACT>(h, a, T, last_obs, first_obs, p, q,
                                                                         smem_actor, smem_critic, st);
    }
    return fail(h, "bad kind %d", h->cfg.kind);
}

extern "C" int b200gym_rollout_actor_critic_norm(b200gym_t *h, const float *actor_dev, const float *critic_dev,
                                                 int n_layers, int h1, int h2, int32_t T, const float *noise_dev,
                                                 float *outputs_dev, void *actions_out_dev, float *obs_dev,
                                                 double *reward_dev, uint8_t *terminated_dev, uint8_t *truncated_dev,
                                                 float *final_obs_dev, float *values_dev, float *advantages_dev,
                                                 float gamma, float gamma_lambda, float *last_obs_dev,
                                                 const float *first_obs_dev, void *stream, int activation,
                                                 const double *obs_mean_dev, const double *obs_var_dev, double eps,
                                                 float clip_obs, const double *ret_var_dev, float clip_reward) {
    const char *what = "b200gym_rollout_actor_critic_norm";
    if (!h) return fail(h, "%s: null handle", what);
    if (int rc = norm_args_check(h, what, obs_mean_dev, obs_var_dev, eps, clip_obs)) return rc;
    if (!(clip_reward > 0.0f)) return fail(h, "%s: clip_reward must be above 0, +inf for none (got %g)", what,
                                           (double)clip_reward);
    if (!ret_var_dev && !std::isinf(clip_reward)) return fail(h, "%s: clip_reward needs ret_var_dev", what);
    if (activation != B200GYM_MLP_RELU && activation != B200GYM_MLP_TANH)
        return fail(h, "%s: activation must be B200GYM_MLP_RELU or B200GYM_MLP_TANH (got %d)", what, activation);
    if (n_layers != 1 && n_layers != 2) return fail(h, "%s: n_layers must be 1 or 2 (got %d)", what, n_layers);
    if (h1 < 1 || h1 > kMlpMaxWidth || (n_layers == 2 && (h2 < 1 || h2 > kMlpMaxWidth)))
        return fail(h, "%s: hidden widths must be 1 .. %d (got %d, %d)", what, kMlpMaxWidth, h1, h2);
    if (T < 1) return fail(h, "%s: T must be at least 1 (got %d)", what, T);
    if (!(gamma >= 0.0f && gamma <= 1.0f && gamma_lambda >= 0.0f && gamma_lambda <= 1.0f))
        return fail(h, "%s: gamma and gamma_lambda must be in [0, 1] (got %g, %g)", what, (double)gamma,
                    (double)gamma_lambda);
    if (!actor_dev || !critic_dev || !noise_dev || !outputs_dev || !actions_out_dev || !obs_dev || !reward_dev ||
        !terminated_dev || !truncated_dev || !values_dev || !advantages_dev || !last_obs_dev)
        return fail(h, "%s: null buffer", what);
    if (!final_obs_dev || !h->cfg.autoreset)
        return fail(h, "%s: the truncation bootstrap needs autoreset and final_obs_dev", what);
    const bool box2d = h->is_lunar || h->is_walker;
    if (box2d && !first_obs_dev) return fail(h, "%s: a Box2D env needs first_obs_dev", what);
    if (n_layers == 1) h2 = 0;
    const int64_t K = h->A == 0 ? h->NACT : h->A, D = h->D;
    const int64_t Pa = h2 == 0 ? h1 * D + h1 + K * h1 + K : h1 * D + h1 + (int64_t)h2 * h1 + h2 + K * h2 + K;
    const int64_t Pc = h2 == 0 ? h1 * D + h1 + h1 + 1 : h1 * D + h1 + (int64_t)h2 * h1 + h2 + h2 + 1;
    const bool vec = h1 % 4 == 0;   // as b200gym_rollout_actor_critic
    const ActorCriticArgs p{{{actor_dev, 0, h1, h2, vec ? 1 : 0, nullptr, nullptr, nullptr}, noise_dev, outputs_dev},
                            critic_dev, values_dev, advantages_dev};
    const ObsNormArgs q{obs_mean_dev, obs_var_dev, eps, clip_obs};
    const size_t smem_actor = (size_t)(Pa + 3) / 4 * 16, smem_critic = (size_t)(Pc + 3) / 4 * 16;
    DeviceGuard guard(h->device);
    const StepArgs a = make_args(h, actions_out_dev, obs_dev, reward_dev, terminated_dev, truncated_dev, final_obs_dev);
    cudaStream_t st = (cudaStream_t)stream;
    const int rc =
        activation == B200GYM_MLP_TANH
            ? launch_rollout_actor_critic_norm<B200GYM_MLP_TANH>(h, a, T, last_obs_dev, first_obs_dev, p, q, smem_actor,
                                                                 smem_critic, st)
            : launch_rollout_actor_critic_norm<B200GYM_MLP_RELU>(h, a, T, last_obs_dev, first_obs_dev, p, q, smem_actor,
                                                                 smem_critic, st);
    return rc ? rc : launch_gae_norm(h, a, T, p, gamma, gamma_lambda, ret_var_dev, eps, clip_reward, st);
}

// ---- normalised inputs and observation moments in the closed-loop rollouts (b200gym_rollout_linear_norm,
// b200gym_rollout_mlp_norm) ----
// The checks both entry points add to their calls without normalisation: the statistics (norm_args_check) and the
// moment buffers, both or neither and only in summary mode
static int norm_moments_check(b200gym *h, const char *what, const double *mean, const double *var, double eps,
                              float clip, const double *sum, const double *sumsq, bool summary) {
    if (int rc = norm_args_check(h, what, mean, var, eps, clip)) return rc;
    if ((sum == nullptr) != (sumsq == nullptr))
        return fail(h, "%s: give both obs_sum_dev and obs_sumsq_dev, or neither", what);
    if (sum && !summary)
        return fail(h, "%s: the observation moments need the summary mode (returns_dev, lengths_dev, ended_dev)", what);
    return 0;
}

// launch_rollout_policy_box2d's sequence with the policy reading the normalised rows of its input (q.mean not null:
// a norm_rows_kernel launch before it) and, in summary mode with m.sum not null, obs_moments_kernel folding the raw
// input rows of step t before that step's launches, whose step sequence overwrites them (the one scratch slice)
template <typename Args>
static int launch_rollout_policy_norm_box2d(b200gym *h, const StepArgs &a, int32_t T, float *last_obs,
                                            const float *first_obs, const Args &p,
                                            void (*policy)(const float *, void *, const Args, const double *,
                                                           const uint8_t *, const uint8_t *, int64_t, int32_t, int,
                                                           int),
                                            size_t smem, const ObsNormArgs &q, const ObsMomentArgs &m, bool summary,
                                            cudaStream_t st, const char *kernel, const char *entry) {
    const unsigned blocks = blocks_for(h->n);
    return launch_rollout_policy_box2d(
        h, a, T, last_obs, first_obs, [&](int32_t) { return p; }, policy, smem, summary, st, kernel, entry,
        [&](int32_t t, const float *, const StepArgs &s, bool after) {
            if (after || !m.sum) return 0;
            obs_moments_kernel<<<blocks, kThreads, 0, st>>>(t == 0 ? first_obs : s.obs, p.ended, s.terminated,
                                                            s.truncated, h->n, (int)h->D, t, m);
            return cudaGetLastError() != cudaSuccess ? fail(h, "obs_moments_kernel: launch failed") : 0;
        },
        [&](const float *o) { return q.mean ? launch_norm_rows(h, o, q, st, entry) : o; });
}

template <int KIND>
static int launch_rollout_linear_norm_kind(b200gym *h, const StepArgs &a, int32_t T, float *last_obs,
                                           const LinearPolicyArgs &p, const ObsNormArgs &q, const ObsMomentArgs &m,
                                           bool summary, cudaStream_t st) {
    const unsigned blocks = blocks_for(h->n);
    if (summary) rollout_linear_norm_kernel<KIND, true><<<blocks, kThreads, 0, st>>>(a, T, last_obs, p, q, m);
    else rollout_linear_norm_kernel<KIND, false><<<blocks, kThreads, 0, st>>>(a, T, last_obs, p, q, m);
    CK(h, cudaGetLastError());
    return 0;
}

extern "C" int b200gym_rollout_linear_norm(b200gym_t *h, const float *weight_dev, const float *bias_dev, int per_env,
                                           int32_t T, void *actions_out_dev, float *obs_dev, double *reward_dev,
                                           uint8_t *terminated_dev, uint8_t *truncated_dev, float *final_obs_dev,
                                           double *returns_dev, int32_t *lengths_dev, uint8_t *ended_dev,
                                           float *last_obs_dev, const float *first_obs_dev, void *stream,
                                           const double *obs_mean_dev, const double *obs_var_dev, double eps,
                                           float clip_obs, double *obs_sum_dev, double *obs_sumsq_dev) {
    const char *what = "b200gym_rollout_linear_norm";
    if (!h) return fail(h, "%s: null handle", what);
    const bool summary = returns_dev != nullptr;
    if (int rc = norm_moments_check(h, what, obs_mean_dev, obs_var_dev, eps, clip_obs, obs_sum_dev, obs_sumsq_dev,
                                    summary))
        return rc;
    if (!obs_mean_dev && !obs_sum_dev)   // neither: b200gym_rollout_linear's own checks and kernels
        return b200gym_rollout_linear(h, weight_dev, bias_dev, per_env, T, actions_out_dev, obs_dev, reward_dev,
                                      terminated_dev, truncated_dev, final_obs_dev, returns_dev, lengths_dev, ended_dev,
                                      last_obs_dev, first_obs_dev, stream);
    if (T < 1) return fail(h, "%s: T must be at least 1 (got %d)", what, T);
    if (!weight_dev || !bias_dev || !last_obs_dev) return fail(h, "%s: null buffer", what);
    if (summary ? (!lengths_dev || !ended_dev || actions_out_dev || obs_dev || reward_dev || terminated_dev ||
                   truncated_dev || final_obs_dev)
                : (!actions_out_dev || !obs_dev || !reward_dev || !terminated_dev || !truncated_dev || lengths_dev ||
                   ended_dev))
        return fail(h, "%s: give either the per-step outputs or returns, lengths and ended", what);
    const bool box2d = h->is_lunar || h->is_walker;
    if (box2d && !first_obs_dev) return fail(h, "%s: a Box2D env needs first_obs_dev", what);
    const int64_t K = h->A == 0 ? h->NACT : h->A;
    const LinearPolicyArgs p{weight_dev, bias_dev, per_env ? K * h->D : 0, per_env ? K : 0, returns_dev, lengths_dev,
                             ended_dev};
    const ObsNormArgs q{obs_mean_dev, obs_var_dev, eps, clip_obs};
    const ObsMomentArgs m{obs_sum_dev, obs_sumsq_dev};
    DeviceGuard guard(h->device);
    const StepArgs a = make_args(h, actions_out_dev, obs_dev, reward_dev, terminated_dev, truncated_dev, final_obs_dev);
    cudaStream_t st = (cudaStream_t)stream;
    float *last = last_obs_dev;
    switch (h->cfg.kind) {
    case B200GYM_CARTPOLE: return launch_rollout_linear_norm_kind<B200GYM_CARTPOLE>(h, a, T, last, p, q, m, summary, st);
    case B200GYM_MOUNTAINCAR:
        return launch_rollout_linear_norm_kind<B200GYM_MOUNTAINCAR>(h, a, T, last, p, q, m, summary, st);
    case B200GYM_MOUNTAINCAR_CONT:
        return launch_rollout_linear_norm_kind<B200GYM_MOUNTAINCAR_CONT>(h, a, T, last, p, q, m, summary, st);
    case B200GYM_PENDULUM: return launch_rollout_linear_norm_kind<B200GYM_PENDULUM>(h, a, T, last, p, q, m, summary, st);
    case B200GYM_ACROBOT: return launch_rollout_linear_norm_kind<B200GYM_ACROBOT>(h, a, T, last, p, q, m, summary, st);
    case B200GYM_LUNARLANDER:
        return launch_rollout_policy_norm_box2d(h, a, T, last, first_obs_dev, p, linear_policy_kernel<4, 8, true>, 0, q,
                                                m, summary, st, "linear_policy_kernel", what);
    case B200GYM_LUNARLANDER_CONT:
        return launch_rollout_policy_norm_box2d(h, a, T, last, first_obs_dev, p, linear_policy_kernel<2, 8, false>, 0,
                                                q, m, summary, st, "linear_policy_kernel", what);
    case B200GYM_BIPEDALWALKER:
    case B200GYM_BIPEDALWALKER_HARDCORE:
        return launch_rollout_policy_norm_box2d(h, a, T, last, first_obs_dev, p, linear_policy_kernel<4, 24, false>, 0,
                                                q, m, summary, st, "linear_policy_kernel", what);
    }
    return fail(h, "bad kind %d", h->cfg.kind);
}

template <int KIND, int ACT>
static int launch_rollout_mlp_norm_kind(b200gym *h, const StepArgs &a, int32_t T, float *last_obs,
                                        const MlpPolicyArgs &p, const ObsNormArgs &q, const ObsMomentArgs &m,
                                        bool per_env, size_t smem, bool summary, cudaStream_t st) {
    const unsigned blocks = blocks_for(h->n);
    if (per_env) {
        if (summary) rollout_mlp_norm_kernel<KIND, true, true, ACT><<<blocks, kThreads, 0, st>>>(a, T, last_obs, p, q, m);
        else rollout_mlp_norm_kernel<KIND, false, true, ACT><<<blocks, kThreads, 0, st>>>(a, T, last_obs, p, q, m);
    } else {
        if (summary)
            rollout_mlp_norm_kernel<KIND, true, false, ACT><<<blocks, kThreads, smem, st>>>(a, T, last_obs, p, q, m);
        else rollout_mlp_norm_kernel<KIND, false, false, ACT><<<blocks, kThreads, smem, st>>>(a, T, last_obs, p, q, m);
    }
    CK(h, cudaGetLastError());
    return 0;
}

template <int K, int D, bool DISCRETE, int ACT>
static int launch_rollout_mlp_norm_box2d(b200gym *h, const StepArgs &a, int32_t T, float *last_obs,
                                         const float *first_obs, const MlpPolicyArgs &p, const ObsNormArgs &q,
                                         const ObsMomentArgs &m, bool per_env, size_t smem, bool summary,
                                         cudaStream_t st) {
    return launch_rollout_policy_norm_box2d(h, a, T, last_obs, first_obs, p,
                                            per_env ? mlp_policy_kernel<K, D, DISCRETE, true, ACT>
                                                    : mlp_policy_kernel<K, D, DISCRETE, false, ACT>,
                                            per_env ? 0 : smem, q, m, summary, st, "mlp_policy_kernel",
                                            "b200gym_rollout_mlp_norm");
}

template <int ACT>
static int launch_rollout_mlp_norm(b200gym *h, const StepArgs &a, int32_t T, float *last_obs, const float *first_obs,
                                   const MlpPolicyArgs &p, const ObsNormArgs &q, const ObsMomentArgs &m, bool pe,
                                   size_t smem, bool summary, cudaStream_t st) {
    switch (h->cfg.kind) {
    case B200GYM_CARTPOLE:
        return launch_rollout_mlp_norm_kind<B200GYM_CARTPOLE, ACT>(h, a, T, last_obs, p, q, m, pe, smem, summary, st);
    case B200GYM_MOUNTAINCAR:
        return launch_rollout_mlp_norm_kind<B200GYM_MOUNTAINCAR, ACT>(h, a, T, last_obs, p, q, m, pe, smem, summary, st);
    case B200GYM_MOUNTAINCAR_CONT:
        return launch_rollout_mlp_norm_kind<B200GYM_MOUNTAINCAR_CONT, ACT>(h, a, T, last_obs, p, q, m, pe, smem, summary,
                                                                          st);
    case B200GYM_PENDULUM:
        return launch_rollout_mlp_norm_kind<B200GYM_PENDULUM, ACT>(h, a, T, last_obs, p, q, m, pe, smem, summary, st);
    case B200GYM_ACROBOT:
        return launch_rollout_mlp_norm_kind<B200GYM_ACROBOT, ACT>(h, a, T, last_obs, p, q, m, pe, smem, summary, st);
    case B200GYM_LUNARLANDER:
        return launch_rollout_mlp_norm_box2d<4, 8, true, ACT>(h, a, T, last_obs, first_obs, p, q, m, pe, smem, summary,
                                                              st);
    case B200GYM_LUNARLANDER_CONT:
        return launch_rollout_mlp_norm_box2d<2, 8, false, ACT>(h, a, T, last_obs, first_obs, p, q, m, pe, smem, summary,
                                                               st);
    case B200GYM_BIPEDALWALKER:
    case B200GYM_BIPEDALWALKER_HARDCORE:
        return launch_rollout_mlp_norm_box2d<4, 24, false, ACT>(h, a, T, last_obs, first_obs, p, q, m, pe, smem, summary,
                                                                st);
    }
    return fail(h, "bad kind %d", h->cfg.kind);
}

extern "C" int b200gym_rollout_mlp_norm(b200gym_t *h, const float *params_dev, int per_env, int n_layers, int h1,
                                        int h2, int32_t T, void *actions_out_dev, float *obs_dev, double *reward_dev,
                                        uint8_t *terminated_dev, uint8_t *truncated_dev, float *final_obs_dev,
                                        double *returns_dev, int32_t *lengths_dev, uint8_t *ended_dev,
                                        float *last_obs_dev, const float *first_obs_dev, void *stream, int activation,
                                        const double *obs_mean_dev, const double *obs_var_dev, double eps,
                                        float clip_obs, double *obs_sum_dev, double *obs_sumsq_dev) {
    const char *what = "b200gym_rollout_mlp_norm";
    if (!h) return fail(h, "%s: null handle", what);
    const bool summary = returns_dev != nullptr;
    if (int rc = norm_moments_check(h, what, obs_mean_dev, obs_var_dev, eps, clip_obs, obs_sum_dev, obs_sumsq_dev,
                                    summary))
        return rc;
    if (!obs_mean_dev && !obs_sum_dev)   // neither: b200gym_rollout_mlp_act's own checks and kernels
        return b200gym_rollout_mlp_act(h, params_dev, per_env, n_layers, h1, h2, T, actions_out_dev, obs_dev,
                                       reward_dev, terminated_dev, truncated_dev, final_obs_dev, returns_dev,
                                       lengths_dev, ended_dev, last_obs_dev, first_obs_dev, stream, activation);
    if (activation != B200GYM_MLP_RELU && activation != B200GYM_MLP_TANH)
        return fail(h, "%s: activation must be B200GYM_MLP_RELU or B200GYM_MLP_TANH (got %d)", what, activation);
    if (n_layers != 1 && n_layers != 2) return fail(h, "%s: n_layers must be 1 or 2 (got %d)", what, n_layers);
    if (h1 < 1 || h1 > kMlpMaxWidth || (n_layers == 2 && (h2 < 1 || h2 > kMlpMaxWidth)))
        return fail(h, "%s: hidden widths must be 1 .. %d (got %d, %d)", what, kMlpMaxWidth, h1, h2);
    if (T < 1) return fail(h, "%s: T must be at least 1 (got %d)", what, T);
    if (!params_dev || !last_obs_dev) return fail(h, "%s: null buffer", what);
    if (summary ? (!lengths_dev || !ended_dev || actions_out_dev || obs_dev || reward_dev || terminated_dev ||
                   truncated_dev || final_obs_dev)
                : (!actions_out_dev || !obs_dev || !reward_dev || !terminated_dev || !truncated_dev || lengths_dev ||
                   ended_dev))
        return fail(h, "%s: give either the per-step outputs or returns, lengths and ended", what);
    const bool box2d = h->is_lunar || h->is_walker;
    if (box2d && !first_obs_dev) return fail(h, "%s: a Box2D env needs first_obs_dev", what);
    if (n_layers == 1) h2 = 0;
    const int64_t K = h->A == 0 ? h->NACT : h->A, D = h->D;
    const int64_t P = h2 == 0 ? h1 * D + h1 + K * h1 + K : h1 * D + h1 + (int64_t)h2 * h1 + h2 + K * h2 + K;
    // as b200gym_rollout_mlp_act
    const bool vec = h1 % 4 == 0 && (!per_env || (P % 4 == 0 && reinterpret_cast<uintptr_t>(params_dev) % 16 == 0));
    const MlpPolicyArgs p{params_dev, per_env ? P : 0, h1, h2, vec ? 1 : 0, returns_dev, lengths_dev, ended_dev};
    const ObsNormArgs q{obs_mean_dev, obs_var_dev, eps, clip_obs};
    const ObsMomentArgs m{obs_sum_dev, obs_sumsq_dev};
    const size_t smem = (size_t)(P + 3) / 4 * 16;
    DeviceGuard guard(h->device);
    const StepArgs a = make_args(h, actions_out_dev, obs_dev, reward_dev, terminated_dev, truncated_dev, final_obs_dev);
    cudaStream_t st = (cudaStream_t)stream;
    const bool pe = per_env != 0;
    if (activation == B200GYM_MLP_TANH)
        return launch_rollout_mlp_norm<B200GYM_MLP_TANH>(h, a, T, last_obs_dev, first_obs_dev, p, q, m, pe, smem,
                                                         summary, st);
    return launch_rollout_mlp_norm<B200GYM_MLP_RELU>(h, a, T, last_obs_dev, first_obs_dev, p, q, m, pe, smem, summary,
                                                     st);
}

// ---- per-env wrapper chains (csrc/subenv.cuh) --------------------------------
// envs [first, first + count); a reshaping chain reads obs_in and fin and writes obs / fin_out / fin64, the others
// work in place on obs
__global__ void __launch_bounds__(kThreads) subenv_step_kernel(const SubenvArgs a, int64_t first, int64_t count,
                                                               const float *obs_in, float *obs, double *reward,
                                                               const uint8_t *term, const uint8_t *trunc,
                                                               const float *fin, float *fin_out, double *fin64,
                                                               float *ep_r, int32_t *ep_l) {
    const int64_t k = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (k >= count) return;
    if (a.reshape) subenv_step_env_io(a, first + k, obs_in, obs, reward, term, trunc, fin, fin_out, fin64, ep_r, ep_l);
    else subenv_step_env(a, first + k, obs, reward, term, trunc, fin, fin_out, fin64, ep_r, ep_l);
}

__global__ void __launch_bounds__(kThreads) subenv_reset_kernel(const SubenvArgs a, const uint8_t *mask,
                                                                const float *obs_in, float *obs) {
    const int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= a.n || (mask && !mask[i])) return;
    if (a.reshape) subenv_reset_env_io(a, i, obs_in, obs);
    else subenv_reset_env(a, i, obs);
}

// ClipAction (clip_action.py:31-40) and RescaleAction (rescale_action.py:62-82) in chain order, in float32, before
// the env sees the action
__global__ void __launch_bounds__(kThreads) subenv_action_kernel(const float *in, float *out, int64_t total, int A,
                                                                 const SubenvActions b) {
    const int64_t e = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (e < total) out[e] = subenv_action(b, (int)(e % A), in[e]);
}

static int launch_actions(const b200gym *h, const float *in, float *out, int64_t rows, int A, const SubenvActions &b,
                          cudaStream_t st) {
    const int64_t total = rows * A;
    subenv_action_kernel<<<blocks_for(total), kThreads, 0, st>>>(in, out, total, A, b);
    CK(h, cudaGetLastError());
    return 0;
}

static int launch_subenv_step(b200gym *h, int64_t first, int64_t count, const float *obs_in, float *obs,
                              double *reward, const uint8_t *term, const uint8_t *trunc, const float *fin,
                              float *fin_out, double *fin64, float *ep_r, int32_t *ep_l, cudaStream_t st) {
    subenv_step_kernel<<<blocks_for(count), kThreads, 0, st>>>(h->sub.args, first, count, obs_in, obs, reward, term,
                                                               trunc, fin, fin_out, fin64, ep_r, ep_l);
    CK(h, cudaGetLastError());
    return 0;
}

static int launch_subenv_reset(b200gym *h, const uint8_t *mask, const float *obs_in, float *obs, cudaStream_t st) {
    subenv_reset_kernel<<<blocks_for(h->n), kThreads, 0, st>>>(h->sub.args, mask, obs_in, obs);
    CK(h, cudaGetLastError());
    return 0;
}

extern "C" int b200gym_subenv_set(b200gym_t *h, const b200gym_subenv *chain) {
    if (!h) return fail(h, "b200gym_subenv_set: null handle");
    if (!chain) {
        if (h->host_ready && h->obs_w != h->D) return fail(h, "b200gym_subenv_set: the host buffers are sized for the chain");
        h->sub.on = h->sub.out_f64 = h->sub.episode = false;
        h->sub.act.num = 0;
        return 0;
    }
    if (!h->cfg.autoreset) return fail(h, "b200gym_subenv_set: a wrapper chain needs autoreset");
    if (chain->num_stages < 0 || chain->num_stages > B200GYM_SUBENV_MAX_STAGES)
        return fail(h, "b200gym_subenv_set: %d stages (at most %d)", chain->num_stages, B200GYM_SUBENV_MAX_STAGES);
    SubenvArgs a{};
    a.num_stages = chain->num_stages;
    a.D = h->D;
    a.n = h->n;
    a.obs_stats = chain->obs_stats_dev;
    a.rew_stats = chain->rew_stats_dev;
    a.ep_return = chain->ep_return_dev;
    a.ep_length = chain->ep_length_dev;
    a.history = chain->history_dev;
    a.head = chain->head_dev;
    a.tstep = chain->t_dev;
    if (chain->raw_reward_type < kRewardPy || chain->raw_reward_type > kRewardF32)
        return fail(h, "b200gym_subenv_set: unknown raw reward type %d", chain->raw_reward_type);
    a.raw_reward_type = chain->raw_reward_type;
    a.int_reward_on_fall = chain->int_reward_on_fall != 0;
    unsigned seen = 0;
    for (int s = 0; s < a.num_stages; s++) {
        const int op = chain->op[s];
        if (op < B200GYM_SUB_EPISODE || op > B200GYM_SUB_FLATTEN || (seen >> op & 1u))
            return fail(h, "b200gym_subenv_set: stage %d has an unknown or repeated op %d", s, op);
        seen |= 1u << op;
        if ((op == B200GYM_SUB_NORM_OBS && !a.obs_stats) || (op == B200GYM_SUB_NORM_REWARD && !a.rew_stats) ||
            (op == B200GYM_SUB_EPISODE && (!a.ep_return || !a.ep_length)) ||
            (op == B200GYM_SUB_FRAME_STACK && (!a.history || !a.head)) || (op == B200GYM_SUB_TIME_AWARE && !a.tstep))
            return fail(h, "b200gym_subenv_set: stage %d needs its state buffers", s);
        if (op == B200GYM_SUB_FRAME_STACK &&
            !(chain->p0[s] >= 1.0 && chain->p0[s] <= B200GYM_SUBENV_MAX_STACK && chain->p0[s] == (int)chain->p0[s]))
            return fail(h, "b200gym_subenv_set: FrameStack needs 1 <= num_stack <= %d, got %g", B200GYM_SUBENV_MAX_STACK,
                        chain->p0[s]);
        a.op[s] = op;
        a.p0[s] = chain->p0[s];
        a.p1[s] = chain->p1[s];
    }
    if (!(seen >> B200GYM_SUB_TIME_AWARE & 1u)) a.tstep = nullptr;
    if (!subenv_resolve(a)) return fail(h, "b200gym_subenv_set: the output width %d is too large", a.W);
    if (h->host_ready && h->obs_w != a.W)
        return fail(h, "b200gym_subenv_set: a chain that changes the observation's width (%d -> %d) must be set before "
                    "b200gym_host_buffers", h->D, a.W);
    SubenvActions act{};
    if (chain->num_action_stages < 0 || chain->num_action_stages > B200GYM_SUBENV_MAX_ACTION_STAGES)
        return fail(h, "b200gym_subenv_set: %d action stages", chain->num_action_stages);
    act.num = chain->num_action_stages;
    for (int s = 0; s < act.num; s++) {
        if (chain->action_op[s] != B200GYM_ACT_CLIP && chain->action_op[s] != B200GYM_ACT_RESCALE)
            return fail(h, "b200gym_subenv_set: unknown action op %d", chain->action_op[s]);
        act.op[s] = chain->action_op[s];
        for (int k = 0; k < 4; k++) {
            act.lo[s][k] = chain->action_low[s][k];
            act.hi[s][k] = chain->action_high[s][k];
            act.amin[s][k] = chain->action_min[s][k];
            act.amax[s][k] = chain->action_max[s][k];
        }
    }
    if (act.num == 0 && chain->clip_action) {
        act.num = 1;
        act.op[0] = kActClip;
        for (int k = 0; k < 4; k++) {
            act.lo[0][k] = chain->act_low[k];
            act.hi[0][k] = chain->act_high[k];
        }
    }
    if (act.num && h->A == 0) return fail(h, "b200gym_subenv_set: ClipAction / RescaleAction need a Box action space");
    if (a.reshape && h->sub.final64 && !h->sub.out)
        CK(h, cudaMalloc((void **)&h->sub.out, (size_t)h->n * a.W * sizeof(float)));
    h->sub.args = a;
    h->sub.act = act;
    h->sub.out_f64 = a.out_f64 != 0;
    h->sub.episode = (seen >> B200GYM_SUB_EPISODE & 1u) != 0;
    h->sub.on = true;
    return 0;
}

extern "C" int b200gym_subenv_width(const b200gym_t *h) {
    if (!h) return -1;
    return h->sub.on ? h->sub.args.W : h->D;
}

extern "C" int b200gym_subenv_step_io(b200gym_t *h, const float *obs_in_dev, float *obs_dev, double *reward_dev,
                                      const uint8_t *terminated_dev, const uint8_t *truncated_dev,
                                      const float *final_obs_in_dev, float *final_obs_dev, double *final_obs64_dev,
                                      float *episode_r_dev, int32_t *episode_l_dev, void *stream) {
    if (!h) return fail(h, "b200gym_subenv_step: null handle");
    if (!h->sub.on) return fail(h, "b200gym_subenv_step: no wrapper chain is set");
    if (!obs_in_dev || !obs_dev || !reward_dev || !terminated_dev || !truncated_dev || !final_obs_in_dev ||
        !final_obs_dev || (h->sub.out_f64 && !final_obs64_dev) || (h->sub.episode && (!episode_r_dev || !episode_l_dev)))
        return fail(h, "b200gym_subenv_step: null buffer");
    if (!h->sub.args.reshape && (obs_in_dev != obs_dev || final_obs_in_dev != final_obs_dev))
        return fail(h, "b200gym_subenv_step_io: this chain works in place (obs_in == obs, final_obs_in == final_obs)");
    DeviceGuard guard(h->device);
    return launch_subenv_step(h, 0, h->n, obs_in_dev, obs_dev, reward_dev, terminated_dev, truncated_dev,
                              final_obs_in_dev, final_obs_dev, final_obs64_dev, episode_r_dev, episode_l_dev,
                              (cudaStream_t)stream);
}

extern "C" int b200gym_subenv_step(b200gym_t *h, float *obs_dev, double *reward_dev, const uint8_t *terminated_dev,
                                   const uint8_t *truncated_dev, float *final_obs_dev, double *final_obs64_dev,
                                   float *episode_r_dev, int32_t *episode_l_dev, void *stream) {
    if (h && h->sub.on && h->sub.args.W != h->D)
        return fail(h, "b200gym_subenv_step: the chain changes the observation's width; use b200gym_subenv_step_io");
    return b200gym_subenv_step_io(h, obs_dev, obs_dev, reward_dev, terminated_dev, truncated_dev, final_obs_dev,
                                  final_obs_dev, final_obs64_dev, episode_r_dev, episode_l_dev, stream);
}

extern "C" int b200gym_subenv_reset_io(b200gym_t *h, const uint8_t *mask_dev, const float *obs_in_dev, float *obs_dev,
                                       void *stream) {
    if (!h || !obs_in_dev || !obs_dev) return fail(h, "b200gym_subenv_reset: null argument");
    if (!h->sub.on) return fail(h, "b200gym_subenv_reset: no wrapper chain is set");
    if (!h->sub.args.reshape && obs_in_dev != obs_dev)
        return fail(h, "b200gym_subenv_reset_io: this chain works in place (obs_in == obs)");
    DeviceGuard guard(h->device);
    return launch_subenv_reset(h, mask_dev, obs_in_dev, obs_dev, (cudaStream_t)stream);
}

extern "C" int b200gym_subenv_reset(b200gym_t *h, const uint8_t *mask_dev, float *obs_dev, void *stream) {
    if (h && h->sub.on && h->sub.args.W != h->D)
        return fail(h, "b200gym_subenv_reset: the chain changes the observation's width; use b200gym_subenv_reset_io");
    return b200gym_subenv_reset_io(h, mask_dev, obs_dev, obs_dev, stream);
}

extern "C" int b200gym_subenv_actions(b200gym_t *h, const float *in_dev, float *out_dev, void *stream) {
    if (!h || !in_dev || !out_dev) return fail(h, "b200gym_subenv_actions: null argument");
    if (!h->sub.on || h->sub.act.num == 0) return fail(h, "b200gym_subenv_actions: the chain has no action stage");
    DeviceGuard guard(h->device);
    return launch_actions(h, in_dev, out_dev, h->n, h->A, h->sub.act, (cudaStream_t)stream);
}

extern "C" int b200gym_clip_actions(const float *in_dev, float *out_dev, int64_t n, int act_dim, const float *low_host,
                                    const float *high_host, void *stream) {
    if (!in_dev || !out_dev || !low_host || !high_host || n <= 0 || act_dim < 1 || act_dim > 4)
        return fail(nullptr, "b200gym_clip_actions: bad argument (1 <= act_dim <= 4)");
    const int dev = device_of(out_dev);
    if (dev < 0) return fail(nullptr, "b200gym_clip_actions: out is not a device pointer");
    DeviceGuard guard(dev);
    SubenvActions b{};
    b.num = 1;
    b.op[0] = kActClip;
    for (int k = 0; k < act_dim; k++) {
        b.lo[0][k] = low_host[k];
        b.hi[0][k] = high_host[k];
    }
    return launch_actions(nullptr, in_dev, out_dev, n, act_dim, b, (cudaStream_t)stream);
}

extern "C" int b200gym_subenv_host_buffers(b200gym_t *h, double **final_obs64_out, float **episode_r_out,
                                           int32_t **episode_l_out) {
    if (!h || !final_obs64_out || !episode_r_out || !episode_l_out)
        return fail(h, "b200gym_subenv_host_buffers: null argument");
    DeviceGuard guard(h->device);
    const size_t n = (size_t)h->n;
    const size_t W = (size_t)b200gym_subenv_width(h);
    if (!h->sub.final64) {
        CK(h, cudaHostAlloc((void **)&h->sub.final64, n * W * sizeof(double), cudaHostAllocMapped));
        CK(h, cudaHostAlloc((void **)&h->sub.ep_r, n * sizeof(float), cudaHostAllocMapped));
        CK(h, cudaHostAlloc((void **)&h->sub.ep_l, n * sizeof(int32_t), cudaHostAllocMapped));
        memset(h->sub.final64, 0, n * W * sizeof(double));
        memset(h->sub.ep_r, 0, n * sizeof(float));
        memset(h->sub.ep_l, 0, n * sizeof(int32_t));
        CK(h, cudaHostGetDevicePointer((void **)&h->sub.final64_dev, h->sub.final64, 0));
        CK(h, cudaHostGetDevicePointer((void **)&h->sub.ep_r_dev, h->sub.ep_r, 0));
        CK(h, cudaHostGetDevicePointer((void **)&h->sub.ep_l_dev, h->sub.ep_l, 0));
        CK(h, cudaMalloc((void **)&h->sub.obs, n * h->D * sizeof(float)));
        CK(h, cudaMalloc((void **)&h->sub.fin, n * h->D * sizeof(float)));
        CK(h, cudaMalloc((void **)&h->sub.reward, n * sizeof(double)));
        CK(h, cudaMalloc((void **)&h->sub.term, n));
        CK(h, cudaMalloc((void **)&h->sub.trunc, n));
        if (h->sub.on && h->sub.args.reshape) CK(h, cudaMalloc((void **)&h->sub.out, n * W * sizeof(float)));
    }
    *final_obs64_out = h->sub.final64;
    *episode_r_out = h->sub.ep_r;
    *episode_l_out = h->sub.ep_l;
    return 0;
}

// ---- host-buffer path -------------------------------------------------------
// The staging buffers are page-locked AND mapped into the device's address space: the step kernel writes its
// results straight into host memory (for the classic-control kinds as bulk shared->global copies of 256-env
// tiles, kernel G with the host as its only destination), so the device->host transfer IS the kernel's store
// stream -- no result mirrors in HBM, no separate D2H copies, no compaction pass for the final observations.
static int ensure_host_io(b200gym *h) {
    if (h->host_ready) return 0;
    const size_t n = (size_t)h->n;
    const size_t act_bytes = h->A == 0 ? n * sizeof(int64_t) : n * h->A * sizeof(float);
    h->obs_w = b200gym_subenv_width(h);   // the chain's output width: a chain that changes it is set before this
    const size_t obs_bytes = n * h->obs_w * sizeof(float);
    const unsigned fl = cudaHostAllocMapped;
    for (int k = 0; k < 2; k++) CK(h, cudaStreamCreateWithFlags(&h->hstream[k], cudaStreamNonBlocking));
    CK(h, cudaHostAlloc(&h->hio.actions, act_bytes, fl));
    CK(h, cudaHostAlloc((void **)&h->hio.obs, obs_bytes, fl));
    CK(h, cudaHostAlloc((void **)&h->hio.reward, n * sizeof(double), fl));
    CK(h, cudaHostAlloc((void **)&h->hio.terminated, n, fl));
    CK(h, cudaHostAlloc((void **)&h->hio.truncated, n, fl));
    CK(h, cudaHostAlloc((void **)&h->hio.final_obs, obs_bytes, fl));
    CK(h, cudaHostAlloc((void **)&h->h_invalid, sizeof(unsigned long long), fl));
    memset(h->hio.actions, 0, act_bytes);
    memset(h->hio.final_obs, 0, obs_bytes);
    // device aliases of the mapped host buffers (identical to the host pointers under unified addressing)
    CK(h, cudaHostGetDevicePointer((void **)&h->dio.obs, h->hio.obs, 0));
    CK(h, cudaHostGetDevicePointer((void **)&h->dio.reward, h->hio.reward, 0));
    CK(h, cudaHostGetDevicePointer((void **)&h->dio.terminated, h->hio.terminated, 0));
    CK(h, cudaHostGetDevicePointer((void **)&h->dio.truncated, h->hio.truncated, 0));
    CK(h, cudaHostGetDevicePointer((void **)&h->dio.final_obs, h->hio.final_obs, 0));
    CK(h, cudaMalloc(&h->dio.actions, act_bytes));   // the actions do live in HBM: every env reads its own once
    CK(h, cudaMalloc((void **)&h->d_mask, n));
    CK(h, cudaEventCreateWithFlags(&h->hevent, cudaEventDisableTiming));
    h->host_ready = true;
    return 0;
}

extern "C" int b200gym_host_buffers(b200gym_t *h, b200gym_host_io *out) {
    if (!h || !out) return fail(h, "b200gym_host_buffers: null argument");
    DeviceGuard guard(h->device);
    if (ensure_host_io(h)) return 1;
    *out = h->hio;
    return 0;
}

static size_t action_size(int action_dtype) {
    switch (action_dtype) {
    case B200GYM_ACT_I64: return 8;
    case B200GYM_ACT_I32: return 4;
    case B200GYM_ACT_U8: return 1;
    default: return 4;
    }
}

// enqueue the chunked pipeline; any failure is reported after both streams have drained
static int step_host_enqueue(b200gym *h, const void *actions_host, int action_dtype, bool want_final) {
    const size_t asz = action_size(action_dtype) * (h->A == 0 ? 1 : h->A);
    const int64_t n = h->n;
    int64_t chunks = n >> 18;                       // 2^20 envs -> 4 chunks: H2D of chunk c+1 under the kernel of c
    chunks = chunks < 1 ? 1 : (chunks > 4 ? 4 : chunks);
    if (const char *hc = getenv("B200GYM_HOST_CHUNKS")) {  // tuning runs
        const int v = atoi(hc);
        if (v >= 1 && v <= 64) chunks = v;
    }
    const int64_t per = ((n + chunks - 1) / chunks + kThreads - 1) / kThreads * kThreads;
    const bool chain = h->sub.on;
    StepArgs a = chain ? make_args(h, h->dio.actions, h->sub.obs, h->sub.reward, h->sub.term, h->sub.trunc, h->sub.fin)
                       : make_args(h, h->dio.actions, h->dio.obs, h->dio.reward, h->dio.terminated, h->dio.truncated,
                                   want_final ? h->dio.final_obs : nullptr);
    a.bulk_sink = 1;
    int c = 0;
    for (int64_t lo = 0; lo < n; lo += per, c++) {
        const int64_t cnt = (lo + per < n) ? per : n - lo;
        cudaStream_t st = h->hstream[c & 1];
        CK(h, cudaMemcpyAsync((char *)h->dio.actions + lo * asz, (const char *)actions_host + lo * asz, cnt * asz,
                              cudaMemcpyHostToDevice, st));
        if (h->sub.on && h->sub.act.num) {
            float *act = (float *)h->dio.actions + lo * h->A;
            if (launch_actions(h, act, act, cnt, h->A, h->sub.act, st)) return 1;
        }
        a.first = lo;
        a.count = cnt;
        a.reset_count = h->reset_count ? h->reset_count + (c % kResetSlots) : nullptr;
        a.toi_count = h->toi_count ? h->toi_count + (c % kResetSlots) : nullptr;
        if (launch_step(h, a, action_dtype, st)) return 1;
        if (chain) {   // the chain over this chunk in HBM, then its dense outputs to the staging buffers in bulk
            const size_t W = (size_t)h->obs_w;
            float *out = h->sub.args.reshape ? h->sub.out : h->sub.obs;
            if (launch_subenv_step(h, lo, cnt, h->sub.obs, out, h->sub.reward, h->sub.term, h->sub.trunc, h->sub.fin,
                                   h->dio.final_obs, h->sub.final64_dev, h->sub.ep_r_dev, h->sub.ep_l_dev, st))
                return 1;
            CK(h, cudaMemcpyAsync(h->hio.obs + lo * W, out + lo * W, cnt * W * sizeof(float),
                                  cudaMemcpyDeviceToHost, st));
            CK(h, cudaMemcpyAsync(h->hio.reward + lo, h->sub.reward + lo, cnt * sizeof(double), cudaMemcpyDeviceToHost,
                                  st));
            CK(h, cudaMemcpyAsync(h->hio.terminated + lo, h->sub.term + lo, cnt, cudaMemcpyDeviceToHost, st));
            CK(h, cudaMemcpyAsync(h->hio.truncated + lo, h->sub.trunc + lo, cnt, cudaMemcpyDeviceToHost, st));
        }
    }
    if (c > 1) {  // stream 0 also waits for the chunks of stream 1
        CK(h, cudaEventRecord(h->hevent, h->hstream[1]));
        CK(h, cudaStreamWaitEvent(h->hstream[0], h->hevent, 0));
    }
    // the sticky invalid-action counter rides along (no separate round trip afterwards)
    CK(h, cudaMemcpyAsync(h->h_invalid, h->invalid, sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->hstream[0]));
    CK(h, cudaMemsetAsync(h->invalid, 0, sizeof(unsigned long long), h->hstream[0]));
    return 0;
}

extern "C" int b200gym_step_host(b200gym_t *h, const void *actions_host, int action_dtype, float *obs_host,
                                 double *reward_host, uint8_t *terminated_host, uint8_t *truncated_host,
                                 float *final_obs_host, int64_t *invalid_out) {
    if (!h) return fail(h, "b200gym_step_host: null handle");
    DeviceGuard guard(h->device);
    if (ensure_host_io(h)) return 1;
    if (h->A == 0 ? (action_dtype == B200GYM_ACT_F32) : (action_dtype != B200GYM_ACT_F32))
        return fail(h, "b200gym_step_host: action dtype code %d does not fit this env's action space", action_dtype);
    if (!actions_host) {
        actions_host = h->hio.actions;
        action_dtype = h->A == 0 ? B200GYM_ACT_I64 : B200GYM_ACT_F32;
    }
    // a wrapper chain reads the terminal rows of the finishing envs, and writes the float64 ones to its own staging
    if (h->sub.on && !h->sub.final64)
        return fail(h, "b200gym_step_host: call b200gym_subenv_host_buffers before stepping with a wrapper chain");
    const bool want_final = (final_obs_host != nullptr || h->sub.on) && h->cfg.autoreset;
    const int rc = step_host_enqueue(h, actions_host, action_dtype, want_final);
    // drain both streams whatever happened: nothing may still be writing into host memory when we return
    const cudaError_t e1 = cudaStreamSynchronize(h->hstream[1]), e0 = cudaStreamSynchronize(h->hstream[0]);
    if (rc) return 1;
    if (e0 != cudaSuccess || e1 != cudaSuccess)
        return fail(h, "b200gym_step_host: %s", cudaGetErrorString(e0 != cudaSuccess ? e0 : e1));
    if (invalid_out) *invalid_out = (int64_t)*h->h_invalid;
    *h->invalid_seen = 0ULL;   // reported (and the device counter cleared) with this call
    // results are in the mapped staging buffers; callers that brought their own arrays get a host copy
    const size_t n = (size_t)h->n, osz = sizeof(float) * h->obs_w;
    if (obs_host && obs_host != h->hio.obs) memcpy(obs_host, h->hio.obs, n * osz);
    if (reward_host && reward_host != h->hio.reward) memcpy(reward_host, h->hio.reward, n * sizeof(double));
    if (terminated_host && terminated_host != h->hio.terminated) memcpy(terminated_host, h->hio.terminated, n);
    if (truncated_host && truncated_host != h->hio.truncated) memcpy(truncated_host, h->hio.truncated, n);
    if (want_final && final_obs_host != h->hio.final_obs)   // rows of the envs that finished in this step only
        for (size_t i = 0; i < n; i++)
            if (h->hio.terminated[i] | h->hio.truncated[i])
                memcpy((char *)final_obs_host + i * osz, (const char *)h->hio.final_obs + i * osz, osz);
    return 0;
}

extern "C" int b200gym_reset_host(b200gym_t *h, const uint8_t *mask_host, const double *bounds_host,
                                  float *obs_host) {
    if (!h) return fail(h, "b200gym_reset_host: null handle");
    DeviceGuard guard(h->device);
    if (ensure_host_io(h)) return 1;
    const size_t n = (size_t)h->n;
    cudaStream_t st = h->hstream[0];
    // the reset kernel writes the rows of the (masked) envs straight into the mapped staging buffer; rows of
    // envs that are not reset keep their content
    // (a reshaping chain: the reset rows land in the HBM copy sub.obs, the chain writes the staging rows)
    const size_t osz = sizeof(float) * h->obs_w;
    if (obs_host && obs_host != h->hio.obs && mask_host) memcpy(h->hio.obs, obs_host, n * osz);
    const bool io = h->sub.on && h->sub.args.reshape;
    if (io && !h->sub.obs)
        return fail(h, "b200gym_reset_host: call b200gym_subenv_host_buffers before resetting with a wrapper chain");
    if (mask_host) CK(h, cudaMemcpyAsync(h->d_mask, mask_host, n, cudaMemcpyHostToDevice, st));
    float *raw = io ? h->sub.obs : h->dio.obs;
    int rc = launch_reset(h, mask_host ? h->d_mask : nullptr, bounds_host, raw, st);
    if (!rc && h->sub.on) rc = launch_subenv_reset(h, mask_host ? h->d_mask : nullptr, raw, h->dio.obs, st);
    const cudaError_t e = cudaStreamSynchronize(st);
    if (rc) return 1;
    if (e != cudaSuccess) return fail(h, "b200gym_reset_host: %s", cudaGetErrorString(e));
    if (obs_host && obs_host != h->hio.obs) memcpy(obs_host, h->hio.obs, n * osz);
    return 0;
}

// ---- state access -----------------------------------------------------------
extern "C" int b200gym_get_state(b200gym_t *h, double *state_dev, int32_t *elapsed_dev, uint64_t *rng_dev,
                                 void *stream) {
    if (!h) return fail(h, "b200gym_get_state: null handle");
    DeviceGuard guard(h->device);
    cudaStream_t st = (cudaStream_t)stream;
    if (state_dev) {
        state_get_kernel<<<blocks_for(h->n), kThreads, 0, st>>>(h->state, state_dev, h->n, h->S);
        CK(h, cudaGetLastError());
    }
    if (elapsed_dev)
        CK(h, cudaMemcpyAsync(elapsed_dev, h->elapsed, sizeof(int32_t) * (size_t)h->n, cudaMemcpyDeviceToDevice, st));
    if (rng_dev) CK(h, cudaMemcpyAsync(rng_dev, h->rng, 32 * (size_t)h->n, cudaMemcpyDeviceToDevice, st));
    return 0;
}

extern "C" int b200gym_lunar_get_bodies(b200gym_t *h, float *bodies_dev, int32_t *flags_dev, void *stream) {
    if (!h || !bodies_dev || !flags_dev) return fail(h, "b200gym_lunar_get_bodies: null argument");
    if (!h->is_lunar) return fail(h, "b200gym_lunar_get_bodies: not a LunarLander handle");
    DeviceGuard guard(h->device);
    lunar_bodies_kernel<<<blocks_for(h->n), kThreads, 0, (cudaStream_t)stream>>>(h->lunar_rec, h->elapsed, bodies_dev,
                                                                                 flags_dev, h->n);
    CK(h, cudaGetLastError());
    return 0;
}

extern "C" int b200gym_lunar_wind_idx(b200gym_t *h, int32_t *wind_idx_host, int32_t *torque_idx_host, int set) {
    if (!h || !wind_idx_host || !torque_idx_host) return fail(h, "b200gym_lunar_wind_idx: null argument");
    if (!h->is_lunar) return fail(h, "b200gym_lunar_wind_idx: not a LunarLander handle");
    DeviceGuard guard(h->device);
    int32_t *d = nullptr;
    const size_t bytes = sizeof(int32_t) * (size_t)h->n;
    CK(h, cudaMalloc((void **)&d, 2 * bytes));
    cudaError_t e = cudaSuccess;
    if (set) {
        e = cudaMemcpy(d, wind_idx_host, bytes, cudaMemcpyHostToDevice);
        if (e == cudaSuccess) e = cudaMemcpy(d + h->n, torque_idx_host, bytes, cudaMemcpyHostToDevice);
    }
    if (e == cudaSuccess) {
        lunar_wind_idx_kernel<<<blocks_for(h->n), kThreads>>>(h->lunar_rec, d, d + h->n, h->n, set);
        e = cudaDeviceSynchronize();
    }
    if (e == cudaSuccess && !set) {
        e = cudaMemcpy(wind_idx_host, d, bytes, cudaMemcpyDeviceToHost);
        if (e == cudaSuccess) e = cudaMemcpy(torque_idx_host, d + h->n, bytes, cudaMemcpyDeviceToHost);
    }
    cudaFree(d);
    if (e != cudaSuccess) return fail(h, "b200gym_lunar_wind_idx: %s", cudaGetErrorString(e));
    return 0;
}

extern "C" int b200gym_walker_get_bodies(b200gym_t *h, float *bodies_dev, int32_t *flags_dev, void *stream) {
    if (!h || !bodies_dev || !flags_dev) return fail(h, "b200gym_walker_get_bodies: null argument");
    if (!h->is_walker) return fail(h, "b200gym_walker_get_bodies: not a BipedalWalker handle");
    DeviceGuard guard(h->device);
    walker_bodies_kernel<<<blocks_for(h->n), kThreads, 0, (cudaStream_t)stream>>>(h->lunar_rec, bodies_dev, flags_dev, h->n);
    CK(h, cudaGetLastError());
    return 0;
}

extern "C" int b200gym_walker_get_terrain(b200gym_t *h, float *terrain_dev, float *polys_dev, int32_t *npoly_dev, void *stream) {
    if (!h || !terrain_dev) return fail(h, "b200gym_walker_get_terrain: null argument");
    if (!h->is_walker) return fail(h, "b200gym_walker_get_terrain: not a BipedalWalker handle");
    DeviceGuard guard(h->device);
    walker_terrain_kernel<<<blocks_for(h->n), kThreads, 0, (cudaStream_t)stream>>>(
        h->lunar_rec, terrain_dev, polys_dev, npoly_dev, h->n, h->cfg.kind == B200GYM_BIPEDALWALKER_HARDCORE);
    CK(h, cudaGetLastError());
    return 0;
}

extern "C" int b200gym_set_state(b200gym_t *h, const double *state_dev, const int32_t *elapsed_dev,
                                 const uint64_t *rng_dev, void *stream) {
    if (!h) return fail(h, "b200gym_set_state: null handle");
    DeviceGuard guard(h->device);
    cudaStream_t st = (cudaStream_t)stream;
    if (state_dev) {
        state_set_kernel<<<blocks_for(h->n), kThreads, 0, st>>>(h->state, state_dev, h->n, h->S);
        CK(h, cudaGetLastError());
    }
    if (elapsed_dev)
        CK(h, cudaMemcpyAsync(h->elapsed, elapsed_dev, sizeof(int32_t) * (size_t)h->n, cudaMemcpyDeviceToDevice, st));
    if (rng_dev) CK(h, cudaMemcpyAsync(h->rng, rng_dev, 32 * (size_t)h->n, cudaMemcpyDeviceToDevice, st));
    return 0;
}

// ---- env snapshots ----------------------------------------------------------
static int snap_prepare(b200gym *h, const char *who) {
    if (!h->snap_bad) {
        if (cudaHostAlloc((void **)&h->snap_bad, sizeof(unsigned long long), cudaHostAllocMapped) != cudaSuccess ||
            cudaHostGetDevicePointer((void **)&h->snap_bad_dev, h->snap_bad, 0) != cudaSuccess) {
            if (h->snap_bad) cudaFreeHost(h->snap_bad);
            h->snap_bad = nullptr;
            return fail(h, "%s: cannot allocate the mapped index-error flag: %s", who, cudaGetErrorString(cudaGetLastError()));
        }
        *h->snap_bad = 0ULL;
        CK(h, cudaFuncSetAttribute(snapshot_save_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   kSnapMaxTileBytes + kThreads * 8));
        CK(h, cudaFuncSetAttribute(snapshot_load_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   kSnapMaxTileBytes + 2 * kThreads * 8 + 8));
    }
    return 0;
}

static SnapArgs snap_args(b200gym *h, int *tile, int *row_bytes) {
    const int kind = h->cfg.kind;
    *row_bytes = snap_row_bytes(kind);
    *tile = snap_tile(*row_bytes);
    SnapArgs a;
    a.rng = reinterpret_cast<uint32_t *>(h->rng);
    a.state = reinterpret_cast<uint32_t *>(h->state);
    a.rec = h->lunar_rec;
    a.elapsed = h->elapsed;
    a.flags = h->flags;
    a.n = h->n;
    a.S2 = 2 * h->S;
    a.W = snap_record_words(kind);
    a.chunks = *row_bytes / 16;
    a.tile_log2 = 0;
    while ((1 << a.tile_log2) < *tile) a.tile_log2++;
    a.bad = h->snap_bad_dev;
    return a;
}

static int snap_save(b200gym *h, const int64_t *idx, int64_t m, void *snap, cudaStream_t st) {
    int T, R;
    const SnapArgs a = snap_args(h, &T, &R);
    const unsigned grid = (unsigned)((m + T - 1) / T);
    snapshot_save_kernel<<<grid, kThreads, (size_t)T * R + T * 8, st>>>(a, idx, m, (unsigned char *)snap);
    CK(h, cudaGetLastError());
    return 0;
}

// bad: the index-error flag to raise (null: the handle's own)
static int snap_load(b200gym *h, const void *snap, int64_t snap_rows, const int64_t *row, const int64_t *dst, int64_t m,
                     cudaStream_t st, unsigned long long *bad = nullptr) {
    int T, R;
    SnapArgs a = snap_args(h, &T, &R);
    if (bad) a.bad = bad;
    const unsigned grid = (unsigned)((m + T - 1) / T);
    snapshot_load_kernel<<<grid, kThreads, (size_t)T * R + 2 * T * 8 + 8, st>>>(a, (const unsigned char *)snap, snap_rows,
                                                                              row, dst, m);
    CK(h, cudaGetLastError());
    return 0;
}

static int snap_check_ptr(b200gym *h, const void *snap, const char *who) {
    if (!snap) return fail(h, "%s: null snapshot pointer", who);
    if ((uintptr_t)snap % 128 != 0) return fail(h, "%s: the snapshot base must be 128-byte aligned", who);
    return 0;
}

extern "C" int b200gym_snapshot_save(b200gym_t *h, const int64_t *idx_dev, int64_t m, void *snap_dev, void *stream) {
    if (!h) return fail(h, "b200gym_snapshot_save: null handle");
    if (m < 0 || (!idx_dev && m > h->n)) return fail(h, "b200gym_snapshot_save: bad row count %lld", (long long)m);
    if (m == 0) return 0;
    if (snap_check_ptr(h, snap_dev, "b200gym_snapshot_save")) return 1;
    DeviceGuard guard(h->device);
    if (snap_prepare(h, "b200gym_snapshot_save")) return 1;
    return snap_save(h, idx_dev, m, snap_dev, (cudaStream_t)stream);
}

extern "C" int b200gym_snapshot_load(b200gym_t *h, const void *snap_dev, const int64_t *row_dev, const int64_t *dst_dev,
                                     int64_t m, void *stream) {
    if (!h) return fail(h, "b200gym_snapshot_load: null handle");
    if (m < 0 || (!dst_dev && m > h->n)) return fail(h, "b200gym_snapshot_load: bad row count %lld", (long long)m);
    if (m == 0) return 0;
    if (snap_check_ptr(h, snap_dev, "b200gym_snapshot_load")) return 1;
    DeviceGuard guard(h->device);
    if (snap_prepare(h, "b200gym_snapshot_load")) return 1;
    // the snapshot holds m rows (row_dev indexes into them)
    return snap_load(h, snap_dev, m, row_dev, dst_dev, m, (cudaStream_t)stream);
}

extern "C" int b200gym_clone(b200gym_t *h, const int64_t *src_dev, void *stream) {
    if (!h || !src_dev) return fail(h, "b200gym_clone: null argument");
    DeviceGuard guard(h->device);
    if (snap_prepare(h, "b200gym_clone")) return 1;
    if (!h->snap_scratch) CK(h, cudaMalloc((void **)&h->snap_scratch, (size_t)h->n * snap_row_bytes(h->cfg.kind)));
    cudaStream_t st = (cudaStream_t)stream;
    if (snap_save(h, nullptr, h->n, h->snap_scratch, st)) return 1;
    return snap_load(h, h->snap_scratch, h->n, src_dev, nullptr, h->n, st);
}

extern "C" int b200gym_snapshot_index_error(b200gym_t *h) {
    if (!h) return -1;
    if (!h->snap_bad || *(volatile unsigned long long *)h->snap_bad == 0ULL) return 0;
    *(volatile unsigned long long *)h->snap_bad = 0ULL;
    return 1;
}

// ---- rollouts from snapshot rows (b200gym_rollout_from) ----
// Branch b's T steps from its row (rollout_from_env), one thread per branch.  The thread's byte of s_flags holds the
// branch's copy of the row's flag byte, so that advance_env never touches the handle's flags
template <int KIND, bool STATES>
__global__ void __launch_bounds__(kThreads) rollout_from_kernel(const StepArgs a, const int32_t T,
                                                                const RolloutFromArgs p) {
    __shared__ uint8_t s_flags[kThreads];
    using ActT = typename std::conditional<Env<KIND>::A == 0, long long, float>::type;
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= a.n) return;
    StepArgs c = a;
    c.flags = s_flags;
    rollout_from_env<KIND, ActT, STATES>(c, b, (int)threadIdx.x, T, p);
}

// The Box2D path: fold step t's reward and flags into the summary of every branch (linear_policy_kernel's fold; step
// 0 starts it at 0.0 + reward)
__global__ void __launch_bounds__(kThreads) rollout_from_fold_kernel(const RolloutFromArgs p, int64_t B,
                                                                     const double *reward, const uint8_t *term,
                                                                     const uint8_t *trunc, int32_t t) {
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    if (t == 0) {
        p.returns[b] = 0.0 + reward[b];
        p.lengths[b] = 1;
        p.ended[b] = (term[b] | trunc[b]) != 0;
    } else if (!p.ended[b]) {
        p.returns[b] = p.returns[b] + reward[b];
        p.lengths[b] = t + 1;
        p.ended[b] = (term[b] | trunc[b]) != 0;
    }
}

// ... and, last, zero the outputs of the branches whose row index is out of range (the load skipped them and raised
// the flag): R bytes of end row and D floats of end observation each, when given
__global__ void __launch_bounds__(kThreads) rollout_from_skip_kernel(const RolloutFromArgs p, int64_t B, int R, int D) {
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const int64_t row = p.row_idx[b];
    if (row >= 0 && row < p.n_rows) return;
    p.returns[b] = 0.0;
    p.lengths[b] = 0;
    p.ended[b] = 0;
    if (!p.end_rows) return;
    for (int c = 0; c < R / 16; c++) reinterpret_cast<uint4 *>(p.end_rows + b * R)[c] = make_uint4(0u, 0u, 0u, 0u);
    for (int k = 0; k < D; k++) p.end_obs[b * D + k] = 0.0f;
}

template <int KIND>
static int launch_rollout_from_kind(b200gym *h, const StepArgs &a, int32_t T, const RolloutFromArgs &p,
                                    cudaStream_t st) {
    if (snap_row_bytes(KIND) != classic_row_bytes<KIND>())
        return fail(h, "b200gym_rollout_from: row layout mismatch for kind %d", KIND);
    if (p.end_rows) rollout_from_kernel<KIND, true><<<blocks_for(a.n), kThreads, 0, st>>>(a, T, p);
    else rollout_from_kernel<KIND, false><<<blocks_for(a.n), kThreads, 0, st>>>(a, T, p);
    CK(h, cudaGetLastError());
    return 0;
}

// The handle's scratch batch of at least B envs, created or grown here, with the snapshot rows of p loaded into envs
// [0, B).  nullptr on failure, with h's error set
static b200gym *from_batch_load(b200gym *h, const RolloutFromArgs &p, int64_t B, cudaStream_t st, const char *who) {
    if (!h->from_batch || h->from_batch->n < B) {
        if (h->from_batch) b200gym_destroy(h->from_batch);
        h->from_batch = nullptr;
        b200gym *s = nullptr;
        if (b200gym_create(&h->cfg, B, h->device, &s)) {
            fail(h, "%s: cannot create the scratch batch: %s", who, b200gym_last_error(nullptr));
            return nullptr;
        }
        h->from_batch = s;
        // the envs a bad row index leaves unloaded step from a valid state: seeded (a zero PCG64 record only ever
        // draws zero, on which BipedalWalker's terrain draws never finish), then reset
        const uint32_t seed[4] = {0u, 0u, 0u, 0u};
        if (b200gym_seed_range(s, seed, 0, st) || launch_reset(s, nullptr, nullptr, nullptr, st)) {
            fail(h, "%s: %s", who, s->err.c_str());
            return nullptr;
        }
    }
    b200gym *s = h->from_batch;
    if (snap_prepare(s, who) || snap_load(s, p.rows, p.n_rows, p.row_idx, nullptr, B, st, h->snap_bad_dev)) {
        fail(h, "%s", s->err.c_str());
        return nullptr;
    }
    return s;
}

// A Box2D rollout from rows, composed of what the engine has: the rows loaded into a handle-owned scratch batch of at
// least B envs (envs [0, B) used), the step sequence of launch_step_box2d per step into one slice of outputs, the fold
// after each step, and with end states a save of the scratch batch.  Its steps take milliseconds, so fusing them would
// save nothing measurable.  Invalid actions count in h's counter and bad row indices raise h's flag
static int launch_rollout_from_box2d(b200gym *h, const RolloutFromArgs &p, int64_t B, const void *actions,
                                     int action_dtype, int32_t T, cudaStream_t st) {
    const char *who = "b200gym_rollout_from";
    b200gym *s = from_batch_load(h, p, B, st, who);
    if (!s) return 1;
    const int64_t D = h->D;
    const size_t obs_bytes = ((size_t)B * D * sizeof(float) + 15) / 16 * 16;
    const size_t r_bytes = ((size_t)B * sizeof(double) + 15) / 16 * 16, f_bytes = ((size_t)B + 15) / 16 * 16;
    void *scratch = nullptr;
    CK(h, cudaMallocAsync(&scratch, obs_bytes + r_bytes + 2 * f_bytes, st));
    unsigned char *base = static_cast<unsigned char *>(scratch);
    float *obs = reinterpret_cast<float *>(base);
    double *reward = reinterpret_cast<double *>(base + obs_bytes);
    uint8_t *term = base + obs_bytes + r_bytes, *trunc = term + f_bytes;
    StepArgs a = make_args(s, nullptr, obs, reward, term, trunc, nullptr);
    a.count = B;
    a.invalid = h->invalid;
    a.invalid_seen = h->invalid_seen_dev;
    const size_t act_row = (size_t)B * std::max(h->A, 1) * action_size(action_dtype);
    const unsigned blocks = blocks_for(B);
    int rc = 0;
    for (int32_t t = 0; t < T && !rc; t++) {
        a.actions = static_cast<const unsigned char *>(actions) + (size_t)t * act_row;
        if (launch_step_box2d(s, a, action_dtype, st)) {
            rc = fail(h, "%s", s->err.c_str());
            break;
        }
        rollout_from_fold_kernel<<<blocks, kThreads, 0, st>>>(p, B, reward, term, trunc, t);
        if (cudaGetLastError() != cudaSuccess) rc = fail(h, "%s: rollout_from_fold_kernel launch failed", who);
    }
    if (!rc && p.end_rows) {
        if (snap_save(s, nullptr, B, p.end_rows, st)) rc = fail(h, "%s", s->err.c_str());
        else if (cudaMemcpyAsync(p.end_obs, obs, (size_t)B * D * sizeof(float), cudaMemcpyDeviceToDevice, st))
            rc = fail(h, "%s: copy of the end observations failed", who);
    }
    if (!rc && p.row_idx) {
        rollout_from_skip_kernel<<<blocks, kThreads, 0, st>>>(p, B, snap_row_bytes(h->cfg.kind), (int)D);
        if (cudaGetLastError() != cudaSuccess) rc = fail(h, "%s: rollout_from_skip_kernel launch failed", who);
    }
    cudaFreeAsync(scratch, st);
    return rc;
}

extern "C" int b200gym_rollout_from(b200gym_t *h, const void *snap_rows_dev, int64_t n_rows, const int64_t *row_idx_dev,
                                    int64_t B, const void *actions_dev, int action_dtype, int32_t T,
                                    double *returns_dev, int32_t *lengths_dev, uint8_t *ended_dev, void *end_rows_dev,
                                    float *end_obs_dev, void *stream) {
    if (!h) return fail(h, "b200gym_rollout_from: null handle");
    if (B < 1) return fail(h, "b200gym_rollout_from: B must be at least 1 (got %lld)", (long long)B);
    if (T < 1) return fail(h, "b200gym_rollout_from: T must be at least 1 (got %d)", T);
    if (n_rows < 0 || (!row_idx_dev && n_rows < B))
        return fail(h, "b200gym_rollout_from: %lld rows cannot start %lld branches without row indices",
                    (long long)n_rows, (long long)B);
    if (!actions_dev || !returns_dev || !lengths_dev || !ended_dev)
        return fail(h, "b200gym_rollout_from: null buffer");
    if (!end_rows_dev != !end_obs_dev)
        return fail(h, "b200gym_rollout_from: give both end_rows_dev and end_obs_dev, or neither");
    if (snap_check_ptr(h, snap_rows_dev, "b200gym_rollout_from")) return 1;
    if (end_rows_dev && (uintptr_t)end_rows_dev % 128 != 0)
        return fail(h, "b200gym_rollout_from: end_rows_dev must be 128-byte aligned");
    const int want = h->A == 0 ? B200GYM_ACT_I64 : B200GYM_ACT_F32;
    if (action_dtype != want)
        return fail(h, "b200gym_rollout_from: this env needs %s actions (got dtype code %d)",
                    h->A == 0 ? "int64" : "float32", action_dtype);
    DeviceGuard guard(h->device);
    // the index-error flag only matters when row indices are given
    if (row_idx_dev && snap_prepare(h, "b200gym_rollout_from")) return 1;
    RolloutFromArgs p{static_cast<const unsigned char *>(snap_rows_dev), n_rows, row_idx_dev, returns_dev, lengths_dev,
                      ended_dev, static_cast<unsigned char *>(end_rows_dev), end_obs_dev, h->snap_bad_dev};
    cudaStream_t st = (cudaStream_t)stream;
    if (h->is_lunar || h->is_walker) return launch_rollout_from_box2d(h, p, B, actions_dev, action_dtype, T, st);
    StepArgs a = make_args(h, actions_dev, nullptr, nullptr, nullptr, nullptr, nullptr);
    a.state = nullptr; a.elapsed = nullptr; a.flags = nullptr; a.rng = nullptr; a.lunar_rec = nullptr;   // not h's envs
    a.n = B; a.count = B;
    switch (h->cfg.kind) {
    case B200GYM_CARTPOLE: return launch_rollout_from_kind<B200GYM_CARTPOLE>(h, a, T, p, st);
    case B200GYM_MOUNTAINCAR: return launch_rollout_from_kind<B200GYM_MOUNTAINCAR>(h, a, T, p, st);
    case B200GYM_MOUNTAINCAR_CONT: return launch_rollout_from_kind<B200GYM_MOUNTAINCAR_CONT>(h, a, T, p, st);
    case B200GYM_PENDULUM: return launch_rollout_from_kind<B200GYM_PENDULUM>(h, a, T, p, st);
    case B200GYM_ACROBOT: return launch_rollout_from_kind<B200GYM_ACROBOT>(h, a, T, p, st);
    }
    return fail(h, "bad kind %d", h->cfg.kind);
}

// ---- closed-loop MLP-policy rollouts from snapshot rows (b200gym_rollout_from_mlp) ----
// Branch b's T steps from its row under its MLP policy (rollout_from_mlp_env), one thread per branch: s_flags as
// rollout_from_kernel's, a shared policy staged per CTA as rollout_mlp_kernel's (PER_BRANCH: branch b's row read from
// device memory), and the statistics as rollout_mlp_norm_kernel's (q.mean null: raw inputs).  Launch bounds as
// rollout_mlp_kernel's
template <int KIND, bool STATES, bool PER_BRANCH, int ACT>
__global__ void __launch_bounds__(kThreads, PER_BRANCH ? 1 : 2)
    rollout_from_mlp_kernel(const StepArgs a, const int32_t T, const RolloutFromMlpArgs p, const ObsNormArgs q) {
    __shared__ uint8_t s_flags[kThreads];
    using Src = MlpActions<KIND, true, PER_BRANCH, ACT>;
    constexpr int K = Src::K, D = Src::D;
    __shared__ double mean[D], sd[D];
    if (q.mean) norm_stage<D>(q, mean, sd);
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const float *w;
    if constexpr (PER_BRANCH) {
        __syncthreads();
        w = p.mlp.params + b * p.mlp.stride;
    } else {
        w = mlp_stage(p.mlp.params, mlp_param_count<K, D>(p.mlp.h1, p.mlp.h2));
    }
    if (b >= a.n) return;
    StepArgs c = a;
    c.flags = s_flags;
    rollout_from_mlp_env<KIND, STATES, PER_BRANCH, ACT>(c, b, (int)threadIdx.x, T, w, p, q.mean ? mean : nullptr, sd,
                                                        q.clip);
}

// The Box2D path's step-0 inputs: snapshot observation row row_idx[b] (row b without indices) into obs[b], zeros for a
// branch whose index is out of range (its outputs are zeroed at the end)
__global__ void __launch_bounds__(kThreads) rollout_from_obs_kernel(const float *snap_obs, const RolloutFromArgs p,
                                                                    int64_t B, int D, float *obs) {
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const int64_t row = p.row_idx ? p.row_idx[b] : b;
    const bool ok = row >= 0 && row < p.n_rows;
    for (int k = 0; k < D; k++) obs[b * D + k] = ok ? snap_obs[row * D + k] : 0.0f;
}

// ... and, with rollout_from_skip_kernel, zero the `bytes` bytes of step-0 action of every skipped branch
__global__ void __launch_bounds__(kThreads) rollout_from_first_skip_kernel(const RolloutFromArgs p, int64_t B,
                                                                           unsigned char *first, int bytes) {
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const int64_t row = p.row_idx[b];
    if (row >= 0 && row < p.n_rows) return;
    for (int k = 0; k < bytes; k++) first[b * bytes + k] = 0;
}

template <int KIND, int ACT>
static int launch_rollout_from_mlp_kind(b200gym *h, const StepArgs &a, int32_t T, const RolloutFromMlpArgs &p,
                                        const ObsNormArgs &q, bool per_branch, size_t smem, cudaStream_t st) {
    if (snap_row_bytes(KIND) != classic_row_bytes<KIND>())
        return fail(h, "b200gym_rollout_from_mlp: row layout mismatch for kind %d", KIND);
    const unsigned blocks = blocks_for(a.n);
    const bool states = p.from.end_rows != nullptr;
    if (per_branch) {
        if (states) rollout_from_mlp_kernel<KIND, true, true, ACT><<<blocks, kThreads, 0, st>>>(a, T, p, q);
        else rollout_from_mlp_kernel<KIND, false, true, ACT><<<blocks, kThreads, 0, st>>>(a, T, p, q);
    } else {
        if (states) rollout_from_mlp_kernel<KIND, true, false, ACT><<<blocks, kThreads, smem, st>>>(a, T, p, q);
        else rollout_from_mlp_kernel<KIND, false, false, ACT><<<blocks, kThreads, smem, st>>>(a, T, p, q);
    }
    CK(h, cudaGetLastError());
    return 0;
}

// A Box2D rollout from rows under an MLP policy, composed as launch_rollout_from_box2d's: the rows loaded into the
// scratch batch, the step-0 inputs gathered from the snapshot's observation rows, and per step the policy launch of
// b200gym_rollout_mlp (mlp_policy_kernel) or b200gym_rollout_mlp_noisy (mlp_noisy_policy_kernel, its outputs to a
// scratch slice), after a norm_rows_kernel launch when normalising, then launch_step_box2d and the fold.  Step 0's
// actions are copied out; the end states and skipped branches as launch_rollout_from_box2d's
template <int K, int D, bool DISCRETE, int ACT>
static int launch_rollout_from_mlp_box2d(b200gym *h, const RolloutFromMlpArgs &p, const float *snap_obs, int64_t B,
                                         int32_t T, const ObsNormArgs &q, bool per_branch, size_t smem,
                                         cudaStream_t st) {
    const char *who = "b200gym_rollout_from_mlp";
    b200gym *s = from_batch_load(h, p.from, B, st, who);
    if (!s) return 1;
    const int action_dtype = DISCRETE ? B200GYM_ACT_I64 : B200GYM_ACT_F32;
    const size_t act_bytes = DISCRETE ? sizeof(long long) : (size_t)K * sizeof(float);   // Box kinds: K = A
    auto up16 = [](size_t x) { return (x + 15) / 16 * 16; };
    const size_t obs_bytes = up16((size_t)B * D * sizeof(float)), a_bytes = up16((size_t)B * act_bytes);
    const size_t r_bytes = up16((size_t)B * sizeof(double)), f_bytes = up16((size_t)B);
    const size_t z_bytes = p.noise ? up16((size_t)B * K * sizeof(float)) : 0;
    void *scratch = nullptr;
    CK(h, cudaMallocAsync(&scratch, 3 * obs_bytes + a_bytes + r_bytes + 2 * f_bytes + z_bytes, st));
    unsigned char *base = static_cast<unsigned char *>(scratch);
    float *first_obs = reinterpret_cast<float *>(base), *obs = reinterpret_cast<float *>(base + obs_bytes);
    float *x = reinterpret_cast<float *>(base + 2 * obs_bytes);
    void *actions = base + 3 * obs_bytes;
    double *reward = reinterpret_cast<double *>(base + 3 * obs_bytes + a_bytes);
    uint8_t *term = base + 3 * obs_bytes + a_bytes + r_bytes, *trunc = term + f_bytes;
    float *outputs = reinterpret_cast<float *>(trunc + f_bytes);
    StepArgs a = make_args(s, actions, obs, reward, term, trunc, nullptr);
    a.count = B;
    a.invalid = h->invalid;
    a.invalid_seen = h->invalid_seen_dev;
    const unsigned blocks = blocks_for(B);
    const size_t pol_smem = per_branch ? 0 : smem;
    int rc = 0;
    rollout_from_obs_kernel<<<blocks, kThreads, 0, st>>>(snap_obs, p.from, B, D, first_obs);
    if (cudaGetLastError() != cudaSuccess) rc = fail(h, "%s: rollout_from_obs_kernel launch failed", who);
    for (int32_t t = 0; t < T && !rc; t++) {
        const float *in = t == 0 ? first_obs : obs;
        if (q.mean) {
            norm_rows_kernel<<<blocks_for(B * D), kThreads, 0, st>>>(in, x, B * D, D, q);
            if (cudaGetLastError() != cudaSuccess) {
                rc = fail(h, "norm_rows_kernel: launch failed");
                break;
            }
            in = x;
        }
        if (p.noise) {
            const MlpNoisyArgs r{p.mlp, p.noise + (int64_t)t * B * K, outputs};
            if (per_branch)
                mlp_noisy_policy_kernel<K, D, DISCRETE, true, ACT><<<blocks, kThreads, 0, st>>>(
                    in, actions, r, nullptr, nullptr, nullptr, B, -1, 1, 0);
            else
                mlp_noisy_policy_kernel<K, D, DISCRETE, false, ACT><<<blocks, kThreads, pol_smem, st>>>(
                    in, actions, r, nullptr, nullptr, nullptr, B, -1, 1, 0);
        } else {
            if (per_branch)
                mlp_policy_kernel<K, D, DISCRETE, true, ACT><<<blocks, kThreads, 0, st>>>(
                    in, actions, p.mlp, nullptr, nullptr, nullptr, B, -1, 1, 0);
            else
                mlp_policy_kernel<K, D, DISCRETE, false, ACT><<<blocks, kThreads, pol_smem, st>>>(
                    in, actions, p.mlp, nullptr, nullptr, nullptr, B, -1, 1, 0);
        }
        if (cudaGetLastError() != cudaSuccess) {
            rc = fail(h, "%s: policy launch failed", who);
            break;
        }
        if (t == 0 && cudaMemcpyAsync(p.first_actions, actions, (size_t)B * act_bytes, cudaMemcpyDeviceToDevice, st)) {
            rc = fail(h, "%s: copy of the step-0 actions failed", who);
            break;
        }
        if (launch_step_box2d(s, a, action_dtype, st)) {
            rc = fail(h, "%s", s->err.c_str());
            break;
        }
        rollout_from_fold_kernel<<<blocks, kThreads, 0, st>>>(p.from, B, reward, term, trunc, t);
        if (cudaGetLastError() != cudaSuccess) rc = fail(h, "%s: rollout_from_fold_kernel launch failed", who);
    }
    if (!rc && p.from.end_rows) {
        if (snap_save(s, nullptr, B, p.from.end_rows, st)) rc = fail(h, "%s", s->err.c_str());
        else if (cudaMemcpyAsync(p.from.end_obs, obs, (size_t)B * D * sizeof(float), cudaMemcpyDeviceToDevice, st))
            rc = fail(h, "%s: copy of the end observations failed", who);
    }
    if (!rc && p.from.row_idx) {
        rollout_from_skip_kernel<<<blocks, kThreads, 0, st>>>(p.from, B, snap_row_bytes(h->cfg.kind), D);
        rollout_from_first_skip_kernel<<<blocks, kThreads, 0, st>>>(p.from, B,
                                                                    static_cast<unsigned char *>(p.first_actions),
                                                                    (int)act_bytes);
        if (cudaGetLastError() != cudaSuccess) rc = fail(h, "%s: skip launch failed", who);
    }
    cudaFreeAsync(scratch, st);
    return rc;
}

template <int ACT>
static int launch_rollout_from_mlp(b200gym *h, const StepArgs &a, int32_t T, const RolloutFromMlpArgs &p,
                                   const float *snap_obs, const ObsNormArgs &q, bool pb, size_t smem, cudaStream_t st) {
    const int64_t B = a.n;
    switch (h->cfg.kind) {
    case B200GYM_CARTPOLE: return launch_rollout_from_mlp_kind<B200GYM_CARTPOLE, ACT>(h, a, T, p, q, pb, smem, st);
    case B200GYM_MOUNTAINCAR: return launch_rollout_from_mlp_kind<B200GYM_MOUNTAINCAR, ACT>(h, a, T, p, q, pb, smem, st);
    case B200GYM_MOUNTAINCAR_CONT:
        return launch_rollout_from_mlp_kind<B200GYM_MOUNTAINCAR_CONT, ACT>(h, a, T, p, q, pb, smem, st);
    case B200GYM_PENDULUM: return launch_rollout_from_mlp_kind<B200GYM_PENDULUM, ACT>(h, a, T, p, q, pb, smem, st);
    case B200GYM_ACROBOT: return launch_rollout_from_mlp_kind<B200GYM_ACROBOT, ACT>(h, a, T, p, q, pb, smem, st);
    case B200GYM_LUNARLANDER:
        return launch_rollout_from_mlp_box2d<4, 8, true, ACT>(h, p, snap_obs, B, T, q, pb, smem, st);
    case B200GYM_LUNARLANDER_CONT:
        return launch_rollout_from_mlp_box2d<2, 8, false, ACT>(h, p, snap_obs, B, T, q, pb, smem, st);
    case B200GYM_BIPEDALWALKER:
    case B200GYM_BIPEDALWALKER_HARDCORE:
        return launch_rollout_from_mlp_box2d<4, 24, false, ACT>(h, p, snap_obs, B, T, q, pb, smem, st);
    }
    return fail(h, "bad kind %d", h->cfg.kind);
}

extern "C" int b200gym_rollout_from_mlp(b200gym_t *h, const void *snap_rows_dev, const float *snap_obs_dev,
                                        int64_t n_rows, const int64_t *row_idx_dev, int64_t B, const float *params_dev,
                                        int per_branch, int n_layers, int h1, int h2, int32_t T, const float *noise_dev,
                                        int activation, const double *obs_mean_dev, const double *obs_var_dev,
                                        double eps, float clip_obs, double *returns_dev, int32_t *lengths_dev,
                                        uint8_t *ended_dev, void *first_actions_dev, void *end_rows_dev,
                                        float *end_obs_dev, void *stream) {
    const char *what = "b200gym_rollout_from_mlp";
    if (!h) return fail(h, "%s: null handle", what);
    if (B < 1) return fail(h, "%s: B must be at least 1 (got %lld)", what, (long long)B);
    if (T < 1) return fail(h, "%s: T must be at least 1 (got %d)", what, T);
    if (n_rows < 0 || (!row_idx_dev && n_rows < B))
        return fail(h, "%s: %lld rows cannot start %lld branches without row indices", what, (long long)n_rows,
                    (long long)B);
    if (activation != B200GYM_MLP_RELU && activation != B200GYM_MLP_TANH)
        return fail(h, "%s: activation must be B200GYM_MLP_RELU or B200GYM_MLP_TANH (got %d)", what, activation);
    if (n_layers != 1 && n_layers != 2) return fail(h, "%s: n_layers must be 1 or 2 (got %d)", what, n_layers);
    if (h1 < 1 || h1 > kMlpMaxWidth || (n_layers == 2 && (h2 < 1 || h2 > kMlpMaxWidth)))
        return fail(h, "%s: hidden widths must be 1 .. %d (got %d, %d)", what, kMlpMaxWidth, h1, h2);
    if (int rc = norm_args_check(h, what, obs_mean_dev, obs_var_dev, eps, clip_obs)) return rc;
    if (noise_dev && per_branch && obs_mean_dev)
        return fail(h, "%s: normalised inputs with noise need one policy shared by every branch (per_branch = 0)", what);
    if (!params_dev || !returns_dev || !lengths_dev || !ended_dev || !first_actions_dev)
        return fail(h, "%s: null buffer", what);
    if (!end_rows_dev != !end_obs_dev) return fail(h, "%s: give both end_rows_dev and end_obs_dev, or neither", what);
    if (snap_check_ptr(h, snap_rows_dev, what)) return 1;
    if (end_rows_dev && (uintptr_t)end_rows_dev % 128 != 0) return fail(h, "%s: end_rows_dev must be 128-byte aligned", what);
    const bool box2d = h->is_lunar || h->is_walker;
    if (box2d && !snap_obs_dev) return fail(h, "%s: a Box2D env needs snap_obs_dev", what);
    if (n_layers == 1) h2 = 0;
    const int64_t K = h->A == 0 ? h->NACT : h->A, D = h->D;
    const int64_t P = h2 == 0 ? h1 * D + h1 + K * h1 + K : h1 * D + h1 + (int64_t)h2 * h1 + h2 + K * h2 + K;
    // as b200gym_rollout_mlp_act
    const bool vec = h1 % 4 == 0 && (!per_branch || (P % 4 == 0 && reinterpret_cast<uintptr_t>(params_dev) % 16 == 0));
    DeviceGuard guard(h->device);
    if (row_idx_dev && snap_prepare(h, what)) return 1;
    const RolloutFromMlpArgs p{{static_cast<const unsigned char *>(snap_rows_dev), n_rows, row_idx_dev, returns_dev,
                                lengths_dev, ended_dev, static_cast<unsigned char *>(end_rows_dev), end_obs_dev,
                                h->snap_bad_dev},
                               {params_dev, per_branch ? P : 0, h1, h2, vec ? 1 : 0, nullptr, nullptr, nullptr},
                               noise_dev,
                               first_actions_dev};
    const ObsNormArgs q{obs_mean_dev, obs_var_dev, eps, clip_obs};
    const size_t smem = (size_t)(P + 3) / 4 * 16;
    cudaStream_t st = (cudaStream_t)stream;
    StepArgs a = make_args(h, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr);
    a.state = nullptr; a.elapsed = nullptr; a.flags = nullptr; a.rng = nullptr; a.lunar_rec = nullptr;   // not h's envs
    a.n = B; a.count = B;
    const bool pb = per_branch != 0;
    if (activation == B200GYM_MLP_TANH)
        return launch_rollout_from_mlp<B200GYM_MLP_TANH>(h, a, T, p, snap_obs_dev, q, pb, smem, st);
    return launch_rollout_from_mlp<B200GYM_MLP_RELU>(h, a, T, p, snap_obs_dev, q, pb, smem, st);
}
