// subenv.cuh -- per-env wrapper chains (`gym.vector.make(id, n, wrappers=[...])`) after the step.
//
// In the reference every sub-env of a SyncVectorEnv carries its own wrapper stack: one RunningMeanStd per env,
// updated with a batch of one, episode accumulators per env, and an autoreset that goes through the outermost
// wrapper, so a finishing env feeds its terminal AND its reset observation to its statistics in the same step
// (gym/vector/sync_vector_env.py:152-156).  Every operation is elementwise (one IEEE add, multiply, divide, sqrt or
// compare per value, no reduction across envs), so the chain runs as one thread per env and is bit-identical to the
// reference.  The stage list travels by value; its branches are uniform across the grid.
//
// Per-env state, SoA float64 rows of n (caller-owned device memory):
//   obs_stats  [2D + 1][n]  NormalizeObservation: mean[D], var[D], count
//   rew_stats  [4][n]       NormalizeReward: mean, var, count, discounted return
//   ep_return  float32 [n], ep_length int32 [n]  RecordEpisodeStatistics accumulators
//
// Chains with FrameStack, TimeAwareObservation or FlattenObservation (`reshape`) change the observation's width and
// dtype along the chain: the step's D float32 values go in, W values come out, and the host resolves the width
// (`width[s]`) and dtype (`f64[s]`) at the input of every stage.  Such a chain reads its input rows and writes its
// output rows in separate buffers (in place where W == D), element by element in output order: an output element
// is traced back to its source (an input element, or the `t` that TimeAwareObservation appends) and run forward
// through the stages, so no thread holds a whole row.  Its extra per-env state:
//   obs_stats  [2w + 1][n]  with w = width at NormalizeObservation's position
//   history    [k * wf][n]  FrameStack's frames (wf = width at its input), float32 or float64 as the dtype there,
//                           written as a ring: frame slot j is rows [j * wf, (j + 1) * wf)
//   head       int32 [n]    the slot of the newest frame
//   tstep      int64 [n]    TimeAwareObservation's t
// Chains without those stages keep the in-place path (subenv_obs_rows).
//
// Compiled into b200gym.cu (so with -fmad=false) and, for the CPU suite, by tests/hostsim/subenv.cpp.
#pragma once
#include <cstdint>

namespace bgym {

constexpr int kSubenvMaxStages = 8;   // every observation / reward stage once
constexpr int kSubenvMaxStack = 64;   // FrameStack's num_stack

enum SubenvOp : int32_t {
    kSubEpisode = 0,      // RecordEpisodeStatistics
    kSubNormObs = 1,      // NormalizeObservation(epsilon)
    kSubNormReward = 2,   // NormalizeReward(gamma, epsilon)
    kSubClipObs = 3,      // TransformObservation(lambda o: np.clip(o, lo, hi))
    kSubClipReward = 4,   // TransformReward(lambda r: np.clip(r, lo, hi))
    kSubFrameStack = 5,   // FrameStack(num_stack = p0)
    kSubTimeAware = 6,    // TimeAwareObservation
    kSubFlatten = 7,      // FlattenObservation
};

// the Python type of a reward (NEP 50 decides how the wrappers combine it)
enum SubenvReward : int32_t {
    kRewardPy = 0,    // a Python float or int: a weak scalar
    kRewardF64 = 1,   // np.float64
    kRewardF32 = 2,   // np.float32
};

struct SubenvArgs {
    int32_t num_stages;
    int32_t op[kSubenvMaxStages];
    int32_t raw_reward_type;      // SubenvReward of the env's raw reward
    int32_t int_reward_on_fall;   // 1: a terminated step with reward -100 is a Python int (BipedalWalker's fall,
                                  // bipedal_walker.py:598-600), whatever raw_reward_type says
    double p0[kSubenvMaxStages], p1[kSubenvMaxStages];   // NormObs: eps; NormReward: gamma, eps; Clip*: lo, hi
    int32_t D;
    int64_t n;
    double *obs_stats, *rew_stats;
    float *ep_return;
    int32_t *ep_length;
    // reshaping chains (all zero otherwise)
    int32_t reshape;                   // 1: the chain has FrameStack, TimeAwareObservation or FlattenObservation
    int32_t W;                         // output width
    int32_t out_f64;                   // 1: the output is float64 (the terminal rows go to fin64)
    int32_t fs;                        // FrameStack's stage index, or -1
    int32_t width[kSubenvMaxStages];   // observation width at the input of stage s
    int32_t f64[kSubenvMaxStages];     // 1: the observation is float64 at the input of stage s
    void *history;
    int32_t *head;
    int64_t *tstep;
};

// Action stages, in the order they apply (the outermost wrapper first): ClipAction clips to the space below it,
// RescaleAction maps [amin, amax] onto it (rescale_action.py:62-82), all in float32
constexpr int kSubenvMaxActionStages = 2;
enum SubenvActionOp : int32_t { kActClip = 0, kActRescale = 1 };
struct SubenvActions {
    int32_t num;
    int32_t op[kSubenvMaxActionStages];
    float lo[kSubenvMaxActionStages][4], hi[kSubenvMaxActionStages][4];
    float amin[kSubenvMaxActionStages][4], amax[kSubenvMaxActionStages][4];
};

// np.clip of numpy 2 (NaN propagates; a value equal to a bound is kept as it is)
__host__ __device__ __forceinline__ double np_clip(double x, double lo, double hi) {
    x = x < lo ? lo : x;
    return x > hi ? hi : x;
}
__host__ __device__ __forceinline__ float np_clipf(float x, float lo, float hi) {
    x = x < lo ? lo : x;
    return x > hi ? hi : x;
}

// action column k through the action stages: `low + (high - low) * ((a - min) / (max - min))`, then np.clip to the
// space below, each operation rounded to float32 (the TU's -fmad=false / -ffp-contract=off keep them separate)
__host__ __device__ __forceinline__ float subenv_action(const SubenvActions &b, int k, float x) {
    for (int s = 0; s < b.num; s++) {
        const float lo = b.lo[s][k], hi = b.hi[s][k];
        if (b.op[s] == kActRescale) x = lo + (hi - lo) * ((x - b.amin[s][k]) / (b.amax[s][k] - b.amin[s][k]));
        x = np_clipf(x, lo, hi);
    }
    return x;
}

// RunningMeanStd.update of one value `x` (normalize.py:18-46, batch of one: batch_mean = x, batch_var =
// (x - x)^2, batch_count = 1), in the order written there; tot = count + 1
__host__ __device__ __forceinline__ void rms_update_one(double x, double bvar, double &mean, double &var, double count,
                                                         double tot) {
    const double delta = x - mean;
    const double new_mean = mean + delta * 1.0 / tot;
    const double m_a = var * count;
    const double m_b = bvar * 1.0;
    const double M2 = m_a + m_b + delta * delta * count * 1.0 / tot;
    mean = new_mean;
    var = M2 / tot;
}

// one observation element through the observation stages in chain order; `mean` / `var` / `count` / `tot` belong
// to the chain's NormalizeObservation (if any)
__host__ __device__ __forceinline__ double subenv_obs_elem(const SubenvArgs &a, double v, double &mean, double &var,
                                                            double count, double tot) {
    for (int s = 0; s < a.num_stages; s++) {
        if (a.op[s] == kSubNormObs) {
            const float x32 = (float)v;                 // the observation is float32 here (np.mean of it is exact)
            const float d32 = x32 - x32;
            rms_update_one(v, (double)(d32 * d32), mean, var, count, tot);
            v = (v - mean) / sqrt(var + a.p0[s]);
        } else if (a.op[s] == kSubClipObs) {
            v = np_clip(v, a.p0[s], a.p1[s]);          // bounds pre-rounded on the host where the obs is float32
        }
    }
    return v;
}

__host__ __device__ __forceinline__ bool subenv_has(const SubenvArgs &a, int op) {
    for (int s = 0; s < a.num_stages; s++)
        if (a.op[s] == op) return true;
    return false;
}

// Observation rows of env i: the terminal row `fin` first when the env finished (written to fin64 as float64 when
// the chain normalises, else to fin_out as float32), then the row `obs` (written back as float32, as
// SyncVectorEnv's concatenate rounds it)
__host__ __device__ __forceinline__ void subenv_obs_rows(const SubenvArgs &a, int64_t i, float *obs, const float *fin,
                                                          float *fin_out, double *fin64, bool done) {
    const int D = a.D;
    const int64_t n = a.n;
    const bool norm = subenv_has(a, kSubNormObs);
    double c0 = 0.0, c1 = 0.0, c2 = 0.0;
    if (norm) {
        c0 = a.obs_stats[2 * D * n + i];
        c1 = c0 + 1.0;
        c2 = c1 + 1.0;
    }
    for (int k = 0; k < D; k++) {
        double mean = 0.0, var = 0.0;
        if (norm) {
            mean = a.obs_stats[k * n + i];
            var = a.obs_stats[(D + k) * n + i];
        }
        double cnt = c0, tot = c1;
        if (done) {
            const double f = subenv_obs_elem(a, (double)fin[i * D + k], mean, var, c0, c1);
            if (norm) fin64[i * D + k] = f;
            else fin_out[i * D + k] = (float)f;
            cnt = c1;
            tot = c2;
        }
        obs[i * D + k] = (float)subenv_obs_elem(a, (double)obs[i * D + k], mean, var, cnt, tot);
        if (norm) {
            a.obs_stats[k * n + i] = mean;
            a.obs_stats[(D + k) * n + i] = var;
        }
    }
    if (norm) a.obs_stats[2 * D * n + i] = done ? c2 : c1;
}

// The step of env i: the reward through the reward stages and RecordEpisodeStatistics, then the observation rows.
// The terminal rows of finishing envs are read from fin and written to fin_out (float32) or fin64 (float64); with
// fin_out == fin and no observation stage they are left where they are
__host__ __device__ __forceinline__ void subenv_step_env(const SubenvArgs &a, int64_t i, float *obs, double *reward,
                                                          const uint8_t *term, const uint8_t *trunc, const float *fin,
                                                          float *fin_out, double *fin64, float *ep_r, int32_t *ep_l) {
    const int64_t n = a.n;
    const bool done = (term[i] | trunc[i]) != 0;
    double r = reward[i];
    int rtype = a.raw_reward_type;
    if (a.int_reward_on_fall && term[i] && r == -100.0) rtype = kRewardPy;
    for (int s = 0; s < a.num_stages; s++) {
        const int op = a.op[s];
        if (op == kSubNormReward) {
            double mean = a.rew_stats[i], var = a.rew_stats[n + i];
            const double count = a.rew_stats[2 * n + i];
            const double ret = a.rew_stats[3 * n + i] * a.p0[s] + r;
            const double d = ret - ret;
            const double tot = count + 1.0;
            rms_update_one(ret, d * d, mean, var, count, tot);
            r = r / sqrt(var + a.p1[s]);
            rtype = kRewardF64;
            a.rew_stats[i] = mean;
            a.rew_stats[n + i] = var;
            a.rew_stats[2 * n + i] = tot;
            a.rew_stats[3 * n + i] = done ? 0.0 : ret;
        } else if (op == kSubClipReward) {
            // np.clip of an np.float32 with Python-float bounds stays float32 (bounds rounded to float32); of a
            // Python number or an np.float64 it is an np.float64
            if (rtype == kRewardF32) {
                r = np_clip(r, (double)(float)a.p0[s], (double)(float)a.p1[s]);
            } else {
                r = np_clip(r, a.p0[s], a.p1[s]);
                rtype = kRewardF64;
            }
        } else if (op == kSubEpisode) {
            // `episode_returns += reward` on a float32 array: a Python number is weak (rounded to float32, float32
            // add), an np.float32 adds in float32, an np.float64 adds in float64 and the sum is rounded
            const double add = rtype == kRewardF64 ? r : (double)(float)r;
            const float acc = (float)((double)a.ep_return[i] + add);
            const int32_t len = a.ep_length[i] + 1;
            if (done) {
                ep_r[i] = acc;
                ep_l[i] = len;
            }
            a.ep_return[i] = done ? 0.0f : acc;
            a.ep_length[i] = done ? 0 : len;
        }
    }
    reward[i] = r;
    if (a.reshape) return;   // subenv_step_env_io writes the observation rows
    if (subenv_has(a, kSubNormObs) || subenv_has(a, kSubClipObs) || fin_out != fin)
        subenv_obs_rows(a, i, obs, fin, fin_out, fin64, done);
}

// reset(): the observation stages on the reset row (NormalizeObservation.reset updates, normalize.py:82-89) and
// RecordEpisodeStatistics.reset's zeroing; NormalizeReward keeps its returns and statistics
__host__ __device__ __forceinline__ void subenv_reset_env(const SubenvArgs &a, int64_t i, float *obs) {
    if (subenv_has(a, kSubEpisode)) {
        a.ep_return[i] = 0.0f;
        a.ep_length[i] = 0;
    }
    if (subenv_has(a, kSubNormObs) || subenv_has(a, kSubClipObs)) subenv_obs_rows(a, i, obs, nullptr, nullptr, nullptr, false);
}

// ---- reshaping chains -------------------------------------------------------------------------------------------
// Host side: the observation's width and dtype at the input of every stage and at the output (a.W, a.out_f64), from
// a.D and the stage list; false when the output is implausibly wide
inline bool subenv_resolve(SubenvArgs &a) {
    int w = a.D, f64 = 0;
    a.fs = -1;
    a.reshape = 0;
    for (int s = 0; s < a.num_stages; s++) {
        a.width[s] = w;
        a.f64[s] = f64;
        switch (a.op[s]) {
        case kSubNormObs: f64 = 1; break;
        case kSubFrameStack: w *= (int)a.p0[s]; a.fs = s; a.reshape = 1; break;
        case kSubTimeAware: w += 1; f64 = 1; a.reshape = 1; break;
        case kSubFlatten: f64 = 0; a.reshape = 1; break;
        default: break;
        }
    }
    a.W = w;
    a.out_f64 = f64;
    return w <= (1 << 20);
}

// The stage where element e at the output of stages [s0, s1) enters: s0 (input element e), or the stage after the
// TimeAwareObservation that appends it as t (np.append(obs, t), time_aware_observation.py:38-47)
__host__ __device__ __forceinline__ int subenv_entry(const SubenvArgs &a, int s0, int s1, int e) {
    int from = s0;
    for (int s = s0; s < s1; s++)
        if (a.op[s] == kSubTimeAware && e == a.width[s]) from = s + 1;
    return from;
}

// element e of one row through stages [from, s1) in the dtype at each position; `cnt` / `tot` are the count of the
// chain's NormalizeObservation before and after this row
__host__ __device__ __forceinline__ double subenv_elem(const SubenvArgs &a, int64_t i, int from, int s1, int e,
                                                        double v, double cnt, double tot) {
    const int64_t n = a.n;
    for (int s = from; s < s1; s++) {
        const int op = a.op[s];
        if (op == kSubNormObs) {
            const int w = a.width[s];
            double mean = a.obs_stats[e * n + i], var = a.obs_stats[(w + e) * n + i];
            double bvar;   // np.var of a batch of one, (x - x)**2 in the observation's dtype
            if (a.f64[s]) {
                const double d = v - v;
                bvar = d * d;
            } else {
                const float x32 = (float)v;
                const float d32 = x32 - x32;
                bvar = (double)(d32 * d32);
            }
            rms_update_one(v, bvar, mean, var, cnt, tot);
            a.obs_stats[e * n + i] = mean;
            a.obs_stats[(w + e) * n + i] = var;
            v = (v - mean) / sqrt(var + a.p0[s]);
        } else if (op == kSubClipObs) {
            v = np_clip(v, a.p0[s], a.p1[s]);   // bounds pre-rounded on the host where the obs is float32
        } else if (op == kSubFlatten) {
            v = (double)(float)v;               // np.asarray(x, dtype=space.dtype): the spaces are float32
        }
    }
    return v;
}

__host__ __device__ __forceinline__ double subenv_hist_get(const SubenvArgs &a, bool f64, int64_t r, int64_t i) {
    return f64 ? ((const double *)a.history)[r * a.n + i] : (double)((const float *)a.history)[r * a.n + i];
}
__host__ __device__ __forceinline__ void subenv_hist_put(const SubenvArgs &a, bool f64, int64_t r, int64_t i, double v) {
    if (f64) ((double *)a.history)[r * a.n + i] = v;
    else ((float *)a.history)[r * a.n + i] = (float)v;
}

// One observation row of env i through every stage: `in` (D float32 values) with TimeAwareObservation's t = `t`.
// `fill`: a reset row, which FrameStack appends num_stack times.  The W outputs go to out32 (rounded to float32, as
// SyncVectorEnv's buffer rounds them) or, when out64 is set, to out64
__host__ __device__ __forceinline__ void subenv_row_io(const SubenvArgs &a, int64_t i, const float *in, int64_t t,
                                                        bool fill, float *out32, double *out64) {
    const int64_t n = a.n;
    const int ns = a.num_stages;
    int norm = -1;
    for (int s = 0; s < ns; s++)
        if (a.op[s] == kSubNormObs) norm = s;
    double cnt = 0.0, tot = 0.0;
    int64_t crow = 0;
    if (norm >= 0) {
        crow = (int64_t)2 * a.width[norm] * n + i;
        cnt = a.obs_stats[crow];
        tot = cnt + 1.0;
    }
    const double tv = (double)t;
    int s1 = ns;   // the stages the output elements run through start after FrameStack
    int wf = 0, k = 1, slot = 0;
    bool hf64 = false;
    if (a.fs >= 0) {
        s1 = a.fs;
        wf = a.width[a.fs];
        k = (int)a.p0[a.fs];
        hf64 = a.f64[a.fs] != 0;
        slot = fill ? 0 : (a.head[i] + 1) % k;
        for (int e = 0; e < wf; e++) {   // the new frame, through the stages below FrameStack, into the ring
            const int from = subenv_entry(a, 0, s1, e);
            const double v = subenv_elem(a, i, from, s1, e, from == 0 ? (double)in[e] : tv, cnt, tot);
            if (fill) {
                for (int j = 0; j < k; j++) subenv_hist_put(a, hf64, (int64_t)j * wf + e, i, v);
            } else {
                subenv_hist_put(a, hf64, (int64_t)slot * wf + e, i, v);
            }
        }
        a.head[i] = slot;
    }
    const int s0 = a.fs >= 0 ? a.fs + 1 : 0;
    for (int e = 0; e < a.W; e++) {
        const int from = subenv_entry(a, s0, ns, e);
        double v;
        if (from != s0) {
            v = tv;
        } else if (a.fs >= 0) {   // frame e / wf of the stack, oldest first: the newest is in `slot`
            const int f = e / wf;
            const int j = (slot + 1 + f) % k;
            v = subenv_hist_get(a, hf64, (int64_t)j * wf + (e - f * wf), i);
        } else {
            v = (double)in[e];
        }
        v = subenv_elem(a, i, from, ns, e, v, cnt, tot);
        if (out64) out64[i * a.W + e] = v;
        else out32[i * a.W + e] = (float)v;
    }
    if (norm >= 0) a.obs_stats[crow] = tot;
}

// The step of env i for a reshaping chain: the reward stages (subenv_step_env), then the observation rows from
// obs_in / fin_in (D wide) to obs_out / fin_out or fin64 (W wide).  A finishing env runs its terminal row (t = the
// episode length) and then its reset row (t = 0, FrameStack filled) through every stage
__host__ __device__ __forceinline__ void subenv_step_env_io(const SubenvArgs &a, int64_t i, const float *obs_in,
                                                             float *obs_out, double *reward, const uint8_t *term,
                                                             const uint8_t *trunc, const float *fin_in,
                                                             float *fin_out, double *fin64, float *ep_r,
                                                             int32_t *ep_l) {
    subenv_step_env(a, i, obs_out, reward, term, trunc, fin_in, fin_out, fin64, ep_r, ep_l);
    const bool done = (term[i] | trunc[i]) != 0;
    const int64_t t = a.tstep ? a.tstep[i] + 1 : 0;
    if (done) subenv_row_io(a, i, fin_in + i * a.D, t, false, fin_out, a.out_f64 ? fin64 : nullptr);
    subenv_row_io(a, i, obs_in + i * a.D, done ? 0 : t, done, obs_out, nullptr);
    if (a.tstep) a.tstep[i] = done ? 0 : t;
}

__host__ __device__ __forceinline__ void subenv_reset_env_io(const SubenvArgs &a, int64_t i, const float *obs_in,
                                                              float *obs_out) {
    if (subenv_has(a, kSubEpisode)) {
        a.ep_return[i] = 0.0f;
        a.ep_length[i] = 0;
    }
    subenv_row_io(a, i, obs_in + i * a.D, 0, true, obs_out, nullptr);
    if (a.tstep) a.tstep[i] = 0;
}

}  // namespace bgym
