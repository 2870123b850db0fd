// hostsim.cpp -- the device source of the step and reset kernels, compiled for the CPU.
//
// TEST INFRASTRUCTURE (never shipped, never imported by gym_b200/): includes gym_b200/csrc/{rng,envs,lunar,walker,
// per_env}.cuh and box2d_consts.h through tests/hostsim/cuda_shim.h and calls the kernels' own per-env drivers
// (per_env.cuh) with plain loops, in the order the kernels are launched.  tests/test_hostsim_cpu.py compares it bit for
// bit with the C oracle, so the `-m "not gpu"` suite runs the code the kernels run: the drivers (action decode,
// TimeLimit, autoreset, final observations, the parked-env and reset lists of the Box2D tasks), solver, scenes, record
// packing, host-computed constants, numpy-compatible RNG.  What it does not run: the kernels' thread and warp logic
// (indexing, shared-memory tiles and lists, the warp-synchronous TOI rounds) and launch code.
#include "cuda_shim.h"

#include <cstdlib>
#include <type_traits>
#include <vector>

#include "../../gym_b200/csrc/rng.cuh"
#include "../../gym_b200/csrc/envs.cuh"
#include "../../gym_b200/csrc/box2d_consts.h"
#include "../../gym_b200/csrc/b2probe.cuh"
#include "../../gym_b200/csrc/per_env.cuh"

using bgym::Pcg64;

namespace {

struct Sim {
    int kind = 0;            // enum b200gym_kind: 5 lunar, 7 lunar continuous, 6 walker, 8 walker hardcore
    int64_t n = 0;
    int max_steps = 0;
    bool defer = true;       // the product default: parked-env TOI pass and reset pass (false: both inline, as
                             // B200GYM_BOX2D_TOI_DEFER=0 / B200GYM_BOX2D_DEFER=0 select on the device)
    int ranges = 1;          // launch ranges a step is split into, the last one ragged (the host path's chunks)
    lunar::Opts opts{};
    std::vector<uint32_t> rec;       // [words][n]
    std::vector<uint64_t> rng;       // [n][4]
    std::vector<int32_t> elapsed;
    std::vector<int32_t> toi_list, reset_list;   // [n]
    std::vector<uint32_t> toi_mid;               // [kToiMidWords][n]
    int32_t toi_count = 0, reset_count = 0;
    int64_t toi_total = 0, reset_total = 0;      // entries the TOI and reset passes have taken, over all steps
    unsigned long long invalid = 0, invalid_seen = 0;
    bool lunar() const { return kind == 5 || kind == 7; }
    bool hardcore() const { return kind == 8; }
};

bool g_consts_ready = false;
void ensure_consts() {
    if (g_consts_ready) return;
    b2l_host::lunar_consts(lunar::kC);
    b2l_host::walker_consts(walker::kC);
    g_consts_ready = true;
}

// one launch range through the passes launch_step_box2d issues: step pass over the range, TOI pass over the parked
// list, reset pass over the reset list (one lane per "warp": live = 1)
template <typename StepF, typename ToiF, typename ResetF>
void box2d_range(const StepArgs &a, StepF step, ToiF toi, ResetF reset) {
    if (a.toi_list) *a.toi_count = 0;
    if (a.reset_list) *a.reset_count = 0;
    for (int64_t j = 0; j < a.count; j++) step(a, j);
    if (a.toi_list)
        for (int idx = 0; idx < *a.toi_count; idx++) toi(a, idx, 1u);
    if (a.reset_list)
        for (int idx = 0; idx < *a.reset_count; idx++) reset(a, idx);
}

}  // namespace

extern "C" {

void *hs_create(int kind, int64_t n, int max_steps, int wind, double gravity, double wind_power, double turbulence_power,
                int defer, int ranges) {
    if (n <= 0 || kind < 5 || kind > 8 || ranges < 1) return nullptr;
    ensure_consts();
    Sim *S = new Sim();
    S->kind = kind; S->n = n; S->max_steps = max_steps; S->defer = defer != 0; S->ranges = ranges;
    S->opts.continuous = kind == 7; S->opts.wind = wind != 0; S->opts.gravity = (float)gravity;
    S->opts.wind_power = wind_power; S->opts.turbulence_power = turbulence_power;
    const size_t words = S->lunar() ? lunar::kWords : (S->hardcore() ? walker::kWordsHC : walker::kWords);
    S->rec.assign(words * (size_t)n, 0u);
    S->rng.assign(4 * (size_t)n, 0ull);
    S->elapsed.assign((size_t)n, 0);
    S->toi_list.assign((size_t)n, 0);
    S->reset_list.assign((size_t)n, 0);
    S->toi_mid.assign((size_t)kToiMidWords * (size_t)n, 0u);
    return S;
}
void hs_destroy(void *h) { delete (Sim *)h; }

void hs_seed_range(void *h, const uint32_t base[4], int64_t first) {   // seed_range_kernel (+ walker_clear_rng32_kernel)
    Sim &S = *(Sim *)h;
    using bgym::u128;
    const u128 b = ((u128)base[3] << 96) | ((u128)base[2] << 64) | ((u128)base[1] << 32) | (u128)base[0];
    for (int64_t i = 0; i < S.n; i++) {
        const u128 seed = b + (u128)(uint64_t)(first + i);
        const uint32_t ent[4] = {(uint32_t)seed, (uint32_t)(seed >> 32), (uint32_t)(seed >> 64), (uint32_t)(seed >> 96)};
        Pcg64 g;
        bgym::pcg64_from_entropy(g, ent);
        bgym::pcg64_store_full(&S.rng[4 * i], g);
        if (!S.lunar()) { S.rec[(int64_t)walker::W_RNG32 * S.n + i] = 0u; S.rec[(int64_t)(walker::W_RNG32 + 1) * S.n + i] = 0u; }
    }
}

void hs_set_wind_idx(void *h, const int32_t *wind, const int32_t *torque) {
    Sim &S = *(Sim *)h;
    for (int64_t i = 0; i < S.n; i++) {
        S.rec[(int64_t)lunar::W_WIND * S.n + i] = (uint32_t)wind[i];
        S.rec[(int64_t)(lunar::W_WIND + 1) * S.n + i] = (uint32_t)torque[i];
    }
}
void hs_get_wind_idx(void *h, int32_t *wind, int32_t *torque) {
    Sim &S = *(Sim *)h;
    for (int64_t i = 0; i < S.n; i++) {
        wind[i] = (int32_t)S.rec[(int64_t)lunar::W_WIND * S.n + i];
        torque[i] = (int32_t)S.rec[(int64_t)(lunar::W_WIND + 1) * S.n + i];
    }
}

void hs_reset(void *h, float *obs) {   // lunar_reset_kernel / walker_reset_kernel<HC>
    Sim &S = *(Sim *)h;
    uint32_t *rec = S.rec.data();
    int32_t *elapsed = S.elapsed.data();
    uint64_t *rng = S.rng.data();
    for (int64_t i = 0; i < S.n; i++) {
        if (S.lunar()) {
            float o[8];
            lunar_reset_env(rec, elapsed, rng, S.n, i, S.opts, o);
            if (obs) store_row<8>(obs, i, o);
        } else {
            float o[24];
            if (S.hardcore()) walker_reset_env<true>(rec, elapsed, rng, S.n, i, o);
            else walker_reset_env<false>(rec, elapsed, rng, S.n, i, o);
            if (obs) store_row<24>(obs, i, o);
        }
    }
}

// actions: int64 [n] (kind 5) or float32 [n][2] (kind 7) or float32 [n][4] (kinds 6, 8); returns #invalid actions
int64_t hs_step(void *h, const void *actions, float *obs_out, double *reward, uint8_t *term, uint8_t *trunc, float *final_obs) {
    Sim &S = *(Sim *)h;
    StepArgs a{};
    a.rng = S.rng.data();
    a.elapsed = S.elapsed.data();
    a.invalid = &S.invalid;
    a.invalid_seen = &S.invalid_seen;
    a.lunar_rec = S.rec.data();
    a.actions = actions;
    a.obs = obs_out; a.reward = reward; a.terminated = term; a.truncated = trunc; a.final_obs = final_obs;
    a.n = S.n;
    a.max_steps = S.max_steps;
    a.autoreset = 1;
    a.lunar_opts = S.opts;
    if (S.defer) {
        a.toi_list = S.toi_list.data(); a.toi_count = &S.toi_count; a.toi_mid = S.toi_mid.data();
        a.reset_list = S.reset_list.data(); a.reset_count = &S.reset_count;
    }
    S.invalid = 0;
    const int64_t per = (S.n + S.ranges - 1) / S.ranges;
    for (a.first = 0; a.first < S.n; a.first += per) {
        a.count = a.first + per < S.n ? per : S.n - a.first;
        switch (S.kind) {
        case 5: box2d_range(a, lunar_step_env<long long, false>, lunar_toi_env, lunar_reset_list_env); break;
        case 7: box2d_range(a, lunar_step_env<float, true>, lunar_toi_env, lunar_reset_list_env); break;
        case 6: box2d_range(a, walker_step_env<false>, walker_toi_env<false>, walker_reset_list_env<false>); break;
        default: box2d_range(a, walker_step_env<true>, walker_toi_env<true>, walker_reset_list_env<true>); break;
        }
        if (S.defer) { S.toi_total += S.toi_count; S.reset_total += S.reset_count; }
    }
    return (int64_t)S.invalid;
}

// how many envs the TOI pass and the reset pass have taken since hs_create (0 and 0 for the inline configuration)
void hs_list_totals(void *h, int64_t *toi, int64_t *reset) {
    Sim &S = *(Sim *)h;
    *toi = S.toi_total;
    *reset = S.reset_total;
}

// the 200 terrain heights and the hardcore boxes of env i (walker kinds); returns the number of boxes
int hs_walker_terrain(void *h, int64_t i, float *terrain200, float *boxes /* [40][4] */) {
    Sim &S = *(Sim *)h;
    for (int k = 0; k < walker::kTerrain; k++) terrain200[k] = __uint_as_float(S.rec[(int64_t)(walker::W_TERRAIN + k) * S.n + i]);
    const int np = S.hardcore() ? (int)S.rec[(int64_t)walker::W_NPOLY * S.n + i] : 0;
    for (int k = 0; k < 4 * np; k++) boxes[k] = __uint_as_float(S.rec[(int64_t)(walker::W_POLY + k) * S.n + i]);
    return np;
}


// envs whose manifold table ever overflowed (b200gym_box2d_overflows on the device)
int64_t hs_overflows(void *h) {
    Sim &S = *(Sim *)h;
    const int64_t row = S.lunar() ? lunar::W_FLAGS : walker::W_FLAGS;
    int64_t c = 0;
    for (int64_t i = 0; i < S.n; i++) c += (S.rec[row * S.n + i] & b2l::kFlagOverflow) != 0;
    return c;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------------------------
// classic control: the per-env drivers of reset_kernel and kernel A (step_kernel) over Env<KIND> of envs.cuh
// (autoreset mode: TimeLimit counter, same-step reset with the env's own PCG64 stream, final_obs rows)
// ---------------------------------------------------------------------------------------------------------------
namespace {

struct Classic {
    int kind = 0;
    int64_t n = 0;
    int max_steps = 0;
    double param0 = 0.0;
    std::vector<double> state;     // [S][n]
    std::vector<uint64_t> rng;     // [n][4]
    std::vector<int32_t> elapsed;
    std::vector<uint8_t> flags;
    unsigned long long invalid = 0, invalid_seen = 0;
};

template <int KIND>
void classic_reset(Classic &C, const double *bounds, float *obs) {   // launch_reset_kind + reset_kernel
    double lo, hi;
    bgym::Env<KIND>::default_bounds(lo, hi);
    if (bounds) { lo = bounds[0]; hi = bounds[1]; }
    double *state = C.state.data();
    int32_t *elapsed = C.elapsed.data();
    uint8_t *flags = C.flags.data();
    uint64_t *rng = C.rng.data();
    for (int64_t i = 0; i < C.n; i++) reset_env_bounded<KIND>(state, elapsed, flags, rng, obs, C.n, i, lo, hi);
}

// kernel A over the whole batch: advance_env for every env, then reset_env for those whose episode ended
template <int KIND>
int64_t classic_step(Classic &C, const void *actions, float *obs_out, double *reward, uint8_t *term, uint8_t *trunc,
                     float *final_obs) {
    using E = bgym::Env<KIND>;
    using ActT = typename std::conditional<E::A == 0, long long, float>::type;
    StepArgs a{};
    a.state = C.state.data(); a.elapsed = C.elapsed.data(); a.flags = C.flags.data(); a.rng = C.rng.data();
    a.invalid = &C.invalid; a.invalid_seen = &C.invalid_seen;
    a.actions = actions;
    a.obs = obs_out; a.reward = reward; a.terminated = term; a.truncated = trunc; a.final_obs = final_obs;
    a.n = C.n; a.first = 0; a.count = C.n;
    a.max_steps = C.max_steps; a.autoreset = 1; a.param0 = C.param0;
    const DirectSinkT<false> sink{a};
    C.invalid = 0;
    std::vector<int64_t> resets;
    for (int64_t i = 0; i < C.n; i++) {
        double s[E::S];
        for (int k = 0; k < E::S; k++) s[k] = a.state[k * a.n + i];
        long long action_int = 0;
        float a0 = 0.0f;
        decode_action<KIND>(__ldg(reinterpret_cast<const ActT *>(a.actions) + i), action_int, a0);
        if (advance_env<KIND>(a, sink, i, s, a.elapsed[i], action_int, a0)) resets.push_back(i);
    }
    for (const int64_t i : resets) reset_env<KIND>(a, sink, i);
    return (int64_t)C.invalid;
}

}  // namespace

extern "C" {

void *hs_classic_create(int kind, int64_t n, int max_steps, double param0) {
    if (n <= 0 || kind < 0 || kind > 4) return nullptr;
    Classic *C = new Classic();
    C->kind = kind; C->n = n; C->max_steps = max_steps; C->param0 = param0;
    C->state.assign(4 * (size_t)n, 0.0);
    C->rng.assign(4 * (size_t)n, 0ull);
    C->elapsed.assign((size_t)n, 0);
    C->flags.assign((size_t)n, 0);
    return C;
}
void hs_classic_destroy(void *h) { delete (Classic *)h; }

void hs_classic_seed_range(void *h, const uint32_t base[4], int64_t first) {
    Classic &C = *(Classic *)h;
    using bgym::u128;
    const u128 b = ((u128)base[3] << 96) | ((u128)base[2] << 64) | ((u128)base[1] << 32) | (u128)base[0];
    for (int64_t i = 0; i < C.n; i++) {
        const u128 seed = b + (u128)(uint64_t)(first + i);
        const uint32_t ent[4] = {(uint32_t)seed, (uint32_t)(seed >> 32), (uint32_t)(seed >> 64), (uint32_t)(seed >> 96)};
        Pcg64 g;
        bgym::pcg64_from_entropy(g, ent);
        bgym::pcg64_store_full(&C.rng[4 * i], g);
    }
}

void hs_classic_reset(void *h, const double *bounds, float *obs) {
    Classic &C = *(Classic *)h;
    switch (C.kind) {
    case 0: classic_reset<B200GYM_CARTPOLE>(C, bounds, obs); break;
    case 1: classic_reset<B200GYM_MOUNTAINCAR>(C, bounds, obs); break;
    case 2: classic_reset<B200GYM_MOUNTAINCAR_CONT>(C, bounds, obs); break;
    case 3: classic_reset<B200GYM_PENDULUM>(C, bounds, obs); break;
    default: classic_reset<B200GYM_ACROBOT>(C, bounds, obs); break;
    }
}

int64_t hs_classic_step(void *h, const void *actions, float *obs, double *reward, uint8_t *term, uint8_t *trunc,
                        float *final_obs) {
    Classic &C = *(Classic *)h;
    switch (C.kind) {
    case 0: return classic_step<B200GYM_CARTPOLE>(C, actions, obs, reward, term, trunc, final_obs);
    case 1: return classic_step<B200GYM_MOUNTAINCAR>(C, actions, obs, reward, term, trunc, final_obs);
    case 2: return classic_step<B200GYM_MOUNTAINCAR_CONT>(C, actions, obs, reward, term, trunc, final_obs);
    case 3: return classic_step<B200GYM_PENDULUM>(C, actions, obs, reward, term, trunc, final_obs);
    default: return classic_step<B200GYM_ACROBOT>(C, actions, obs, reward, term, trunc, final_obs);
    }
}

void hs_classic_get_state(void *h, double *state_aos /* [n][S] */, int S) {
    Classic &C = *(Classic *)h;
    for (int64_t i = 0; i < C.n; i++)
        for (int k = 0; k < S; k++) state_aos[i * S + k] = C.state[(int64_t)k * C.n + i];
}

// CartPole's small-angle sin/cos kernel alone (csrc/envs.cuh: sincos_small)
void hs_sincos_small(const double *x, int64_t n, double *sn, double *cs) {
    for (int64_t i = 0; i < n; i++) bgym::sincos_small(x[i], sn[i], cs[i]);
}


// glibc_trig.cuh: the restated glibc sin / cos, evaluated by the host build of the device header
void hs_glibc_trig(const double *x, int64_t n, double *sn, double *cs) {
    for (int64_t i = 0; i < n; i++) { sn[i] = bgym::gt::sin(x[i]); cs[i] = bgym::gt::cos(x[i]); }
}
// arguments in [lo, hi) (splitmix64 stream) where gt::sq(x) differs bitwise from libm pow(x, 2.0); *neq_out counts
// those where pow(x, 2.0) itself differs from x * x (why the restatement exists)
int64_t hs_glibc_sq_mismatches(uint64_t seed, int64_t n, double lo, double hi, int64_t *neq_out) {
    int64_t bad = 0, neq = 0;
    uint64_t st = seed;
    volatile double two = 2.0;   // keep the compiler from folding pow(x, 2.0) into x * x
    for (int64_t i = 0; i < n; i++) {
        uint64_t z = (st += 0x9E3779B97F4A7C15ULL);
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
        z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
        z ^= z >> 31;
        const double x = lo + (hi - lo) * ((double)(z >> 11) * (1.0 / 9007199254740992.0));
        const double a = std::pow(x, two), b = bgym::gt::sq(x), c = x * x;
        bad += std::memcmp(&a, &b, 8) != 0;
        neq += std::memcmp(&a, &c, 8) != 0;
    }
    if (neq_out) *neq_out = neq;
    return bad;
}

// number of arguments in [lo, hi) (splitmix64 stream) where sin or cos differs bitwise from this process's libm
int64_t hs_glibc_trig_mismatches(uint64_t seed, int64_t n, double lo, double hi) {
    int64_t bad = 0;
    uint64_t st = seed;
    for (int64_t i = 0; i < n; i++) {
        uint64_t z = (st += 0x9E3779B97F4A7C15ULL);
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
        z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
        z ^= z >> 31;
        const double x = lo + (hi - lo) * ((double)(z >> 11) * (1.0 / 9007199254740992.0));
        const double a = std::sin(x), b = bgym::gt::sin(x), c = std::cos(x), d = bgym::gt::cos(x);
        bad += (std::memcmp(&a, &b, 8) != 0) + (std::memcmp(&c, &d, 8) != 0);
    }
    return bad;
}


// The device's b2TimeOfImpact and the conservative shortcut in front of it (b2lite_toi.cuh), for one sweep of a
// task polygon (shape 0 = lander, 1 = lander leg, 2 = walker hull, 3 = walker upper leg, 4 = walker lower leg)
// against the static edge v1-v2 or, with `box` set, the axis-aligned box {x0, ylo, x1, yhi}.
// Returns the b2TOIOutput state (3 = touching), *t_out, and *cannot_touch = what toi_cannot_touch says.
int hs_toi_probe(int shape, const float *c0, float a0, const float *c1, float a1, const float *v1, const float *v2,
                 const float *box, float *t_out, int *cannot_touch) {
    ensure_consts();
    const b2l::ShapeConst &sh = shape < 2 ? lunar::kC.shape[shape] : walker::kC.shape[shape - 2];
    b2l::DProxy pA, pB;
    if (box) {
        pA.count = 4;
        pA.v[0] = b2l::V(box[2], box[1]); pA.v[1] = b2l::V(box[2], box[3]); pA.v[2] = b2l::V(box[0], box[3]); pA.v[3] = b2l::V(box[0], box[1]);
    } else {
        pA.count = 2;
        pA.v[0] = b2l::V(v1[0], v1[1]); pA.v[1] = b2l::V(v2[0], v2[1]);
    }
    pB.count = sh.count;
    for (int i = 0; i < sh.count; i++) pB.v[i] = sh.verts[i];
    b2l::Sweep sA, sB;
    sA.localCenter = b2l::V(0.0f, 0.0f); sA.c0 = b2l::V(0.0f, 0.0f); sA.c = b2l::V(0.0f, 0.0f); sA.a0 = 0.0f; sA.a = 0.0f; sA.alpha0 = 0.0f;
    sB.localCenter = sh.localCenter; sB.c0 = b2l::V(c0[0], c0[1]); sB.c = b2l::V(c1[0], c1[1]); sB.a0 = a0; sB.a = a1; sB.alpha0 = 0.0f;
    b2l::xform xf1;
    xf1.q = b2l::rot_of(a1);
    xf1.p = b2l::sub(sB.c, b2l::rmul(xf1.q, sh.localCenter));
    *cannot_touch = b2l::toi_cannot_touch(sh, xf1, sB, pA) ? 1 : 0;
    return b2l::time_of_impact(*t_out, pA, sA, pB, sB, 1.0f);
}

// b200gym_selftest_box2d's per-record dispatch (csrc/b2probe.cuh) over in[n][16] -> out[n][16]
void hs_box2d_probe(int op, const float *in, int64_t n, float *out) {
    ensure_consts();
    for (int64_t i = 0; i < n; i++) b2probe::probe_case(op, in + i * b2probe::kProbeWords, out + i * b2probe::kProbeWords);
}

// The task polygon `shape` as the device constants hold it: vertices (x, y pairs) into out, local centre into lc;
// returns the vertex count.
int hs_shape_verts(int shape, float *out, float *lc) {
    ensure_consts();
    const b2l::ShapeConst &sh = shape < 2 ? lunar::kC.shape[shape] : walker::kC.shape[shape - 2];
    for (int i = 0; i < sh.count; i++) { out[2 * i] = sh.verts[i].x; out[2 * i + 1] = sh.verts[i].y; }
    lc[0] = sh.localCenter.x; lc[1] = sh.localCenter.y;
    return sh.count;
}

}  // extern "C"
