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
// Compiled into b200gym.cu (so with -fmad=false) and, for the CPU suite, by tests/hostsim/subenv.cpp.
#pragma once
#include <cstdint>

namespace bgym {

constexpr int kSubenvMaxStages = 5;

enum SubenvOp : int32_t {
    kSubEpisode = 0,      // RecordEpisodeStatistics
    kSubNormObs = 1,      // NormalizeObservation(epsilon)
    kSubNormReward = 2,   // NormalizeReward(gamma, epsilon)
    kSubClipObs = 3,      // TransformObservation(lambda o: np.clip(o, lo, hi))
    kSubClipReward = 4,   // TransformReward(lambda r: np.clip(r, lo, hi))
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

}  // namespace bgym
