"""numpy restatement of the per-env wrapper chains (gym_b200/subenv.py, csrc/subenv.cuh).  Test infrastructure.

``SubenvChainRef`` takes the RAW outputs of a SyncVectorEnv of unwrapped envs (float32 observations, float64 rewards,
flags, float32 terminal rows) and returns what the same SyncVectorEnv over wrapped envs returns.  It is written
from the reference wrappers with numpy doing the typing, vectorised over envs only where every operation is
elementwise:

* RunningMeanStd.update with a batch of one (gym/wrappers/normalize.py:18-46): batch mean x, batch var (x - x)**2
  in the dtype of x, batch count the int 1, the count a float;
* NormalizeObservation (:73-94): float32 observations in, float64 out; the autoreset runs the terminal and then the
  reset observation of a finishing env through it (gym/vector/sync_vector_env.py:152-156);
* NormalizeReward (:128-144): returns = returns * gamma + [r]; r / sqrt(var + eps) is a float64;
* np.clip with Python-float bounds keeps the dtype of its array argument (NEP 50), and turns a Python float into an
  np.float64;
* RecordEpisodeStatistics (record_episode_statistics.py:103-151): `episode_returns += reward` on a float32 array,
  where a Python-number reward is weak (float32 add) and a numpy scalar is not (add in its dtype, then round).

The Python type of the reward is tracked per env: BipedalWalker's rewards are np.float32 except the -100 of a fall, a
Python int (bipedal_walker.py:598-600).
"""
import numpy as np

# the Python type of the raw reward of each classic-control / Box2D id ("py": a Python float or int)
RAW_REWARD_TYPE = {"CartPole": "py", "MountainCar-": "py", "MountainCarContinuous": "py", "Acrobot": "py",
                   "Pendulum": "f64", "LunarLander": "f64", "BipedalWalker": "f32"}
PY, F64, F32 = 0, 1, 2


def raw_reward_type(env_id):
    for prefix, t in RAW_REWARD_TYPE.items():
        if env_id.startswith(prefix):
            return t
    raise KeyError(env_id)


def _update(mean, var, count, x, batch_var):
    """update_mean_var_count_from_moments(mean, var, count, x, batch_var, 1), in the order written there."""
    batch_count = 1
    delta = x - mean
    tot_count = count + batch_count
    new_mean = mean + delta * batch_count / tot_count
    m_a = var * count
    m_b = batch_var * batch_count
    M2 = m_a + m_b + np.square(delta) * count * batch_count / tot_count
    return new_mean, M2 / tot_count, tot_count


class SubenvChainRef:
    """stages: ``[(name, kwargs), ...]`` innermost first (``gym_b200.subenv`` stage ``describe()`` lists)."""

    def __init__(self, stages, env_id, n, obs_dim):
        self.stages = [(name, dict(kw)) for name, kw in stages]
        self.raw_type = raw_reward_type(env_id)
        self.n, self.d = int(n), int(obs_dim)
        self.obs_mean = np.zeros((n, obs_dim))
        self.obs_var = np.ones((n, obs_dim))
        self.obs_count = np.full((n, 1), 1e-4)
        self.rew_mean, self.rew_var, self.rew_count = np.zeros(n), np.ones(n), np.full(n, 1e-4)
        self.returns = np.zeros(n)
        self.ep_return = np.zeros(n, np.float32)
        self.ep_length = np.zeros(n, np.int32)
        self.normalizes_obs = any(name == "NormalizeObservation" for name, _ in self.stages)

    def _obs_rows(self, rows, x):
        """Observation stages over the rows `rows` (float32 (m, D)), updating their statistics."""
        for name, kw in self.stages:
            if name == "NormalizeObservation":
                assert x.dtype == np.float32
                mean, var, count = _update(self.obs_mean[rows], self.obs_var[rows], self.obs_count[rows], x,
                                           np.square(x - x))
                self.obs_mean[rows], self.obs_var[rows], self.obs_count[rows] = mean, var, count
                x = (x - mean) / np.sqrt(var + kw["epsilon"])
            elif name == "ClipObservation":
                x = np.clip(x, kw["low"], kw["high"])
        return x

    def reset(self, obs):
        """reset(): observation stages with updates; RecordEpisodeStatistics zeroes its accumulators."""
        self.ep_return[:] = 0
        self.ep_length[:] = 0
        return self._obs_rows(np.arange(self.n), np.asarray(obs, np.float32)).astype(np.float32)

    def step(self, obs, reward, terminated, truncated, final_obs):
        """-> obs float32, reward float64, terminal rows (float64 when normalised, else float32; rows of unfinished
        envs are zero), episode return float32 / length int32 (finishing envs only; NaN / -1 elsewhere)."""
        term = np.asarray(terminated, bool)
        done = term | np.asarray(truncated, bool)
        r = np.asarray(reward, np.float64).copy()
        rtype = np.full(self.n, {"py": PY, "f64": F64, "f32": F32}[self.raw_type])
        if self.raw_type == "f32":            # BipedalWalker: `reward = -100` on a fall is a Python int
            rtype[term & (r == -100.0)] = PY
        ep_r = np.full(self.n, np.nan, np.float32)
        ep_l = np.full(self.n, -1, np.int32)
        for name, kw in self.stages:
            if name == "RecordEpisodeStatistics":
                weak = rtype != F64               # Python number: cast to float32; np.float32: float32 add
                self.ep_return[weak] = self.ep_return[weak] + r[weak].astype(np.float32)
                self.ep_return[~weak] = (self.ep_return[~weak] + r[~weak]).astype(np.float32)
                self.ep_length = self.ep_length + np.int32(1)
                ep_r[done], ep_l[done] = self.ep_return[done], self.ep_length[done]
                self.ep_return[done], self.ep_length[done] = 0, 0
            elif name == "NormalizeReward":
                self.returns = self.returns * kw["gamma"] + r
                self.rew_mean, self.rew_var, self.rew_count = _update(
                    self.rew_mean, self.rew_var, self.rew_count, self.returns, np.square(self.returns - self.returns))
                r = r / np.sqrt(self.rew_var + kw["epsilon"])
                self.returns[done] = 0.0
                rtype[:] = F64
            elif name == "ClipReward":
                f32 = rtype == F32                # np.float32 stays float32, bounds rounded; the rest -> np.float64
                r[f32] = np.clip(r[f32].astype(np.float32), kw["low"], kw["high"])
                r[~f32] = np.clip(r[~f32], kw["low"], kw["high"])
                rtype[~f32] = F64
        fin = np.zeros((self.n, self.d), np.float64 if self.normalizes_obs else np.float32)
        rows = np.flatnonzero(done)
        if len(rows):
            fin[rows] = self._obs_rows(rows, np.asarray(final_obs, np.float32)[rows])
        out = self._obs_rows(np.arange(self.n), np.asarray(obs, np.float32)).astype(np.float32)
        return out, r, fin, ep_r, ep_l
