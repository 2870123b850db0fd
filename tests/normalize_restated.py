"""Numpy restatements of NormalizeObservation / NormalizeReward (gym/wrappers/normalize.py:8-144) over a batch.

``Reference``  the reference as it computes: ``np.mean`` / ``np.var`` of the batch as given (float32 observations
               are summed in float32, row by row), the float64 Chan update, float64 outputs.
``Restated64`` what the device normalisers compute: float64 sums of the deviations from the running mean (the
               pivot), the same Chan update, in the kernels' order of operations.
``Restated64.bound`` carries, step by step, a bound on how far the reference's observation statistics and outputs
can be from the float64 ones: the float32 accumulation error of ``np.mean`` / ``np.var`` over the batch,
propagated through the update (a convex combination of the old statistics and the batch's).
"""
import os

import numpy as np

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference", "normalize_wrappers.npz")
EPS = 1e-8
U32 = 2.0 ** -24


def gamma_n(n, u):
    return n * u / (1 - n * u)


def chan(stats, sums, d, bn):
    """update_mean_var_count_from_moments from the pivoted batch sums (pivot = stats' mean), the kernels' order."""
    dm = sums[:d] / bn
    batch_var = sums[d:] / bn - dm * dm
    cnt = stats[2 * d]
    tot = cnt + bn
    mean = stats[:d] + dm * bn / tot
    m2 = stats[d:2 * d] * cnt + batch_var * bn + dm * dm * cnt * bn / tot
    return mean, m2 / tot, tot


def update(stats, sums, d, bn):
    """chan() as one {mean, var, count} vector."""
    mean, var, tot = chan(stats, sums, d, bn)
    return np.concatenate([mean, var, [tot]])


def moments64(x, mean):
    """Pivoted float64 sums of a [n][d] batch: sum(x - mean) and sum((x - mean)^2) per column, pairwise."""
    dev = np.ascontiguousarray((x - mean).T)
    return np.concatenate([np.sum(dev, axis=1), np.sum(dev * dev, axis=1)])


def initial(d):
    """RunningMeanStd() of normalize.py:11-15: mean 0, var 1, count 1e-4, as one {mean, var, count} vector."""
    return np.concatenate([np.zeros(d), np.ones(d), [1e-4]])


class Reference:
    """NormalizeReward(NormalizeObservation(env), gamma) of the reference, fed the rows the env returned."""

    def __init__(self, n, d, gamma):
        self.d, self.gamma = d, gamma
        self.obs_mean, self.obs_var, self.obs_count = np.zeros(d), np.ones(d), 1e-4
        self.ret_mean, self.ret_var, self.ret_count = np.zeros(()), np.ones(()), 1e-4
        self.returns = np.zeros(n)

    @staticmethod
    def _update(mean, var, count, x):
        # normalize.py:18-46, verbatim in numpy
        batch_mean, batch_var, batch_count = np.mean(x, axis=0), np.var(x, axis=0), x.shape[0]
        delta = batch_mean - mean
        tot_count = count + batch_count
        new_mean = mean + delta * batch_count / tot_count
        m_a = var * count
        m_b = batch_var * batch_count
        m2 = m_a + m_b + np.square(delta) * count * batch_count / tot_count
        return new_mean, m2 / tot_count, tot_count

    def normalize(self, obs):
        self.obs_mean, self.obs_var, self.obs_count = self._update(self.obs_mean, self.obs_var, self.obs_count, obs)
        return (obs - self.obs_mean) / np.sqrt(self.obs_var + EPS)

    def reward(self, rews, done):
        self.returns = self.returns * self.gamma + rews
        self.ret_mean, self.ret_var, self.ret_count = self._update(self.ret_mean, self.ret_var, self.ret_count,
                                                                   self.returns)
        out = rews / np.sqrt(self.ret_var + EPS)
        self.returns[done] = 0.0
        return out


class Restated64:
    """The device normalisers in float64 numpy; ``bound(x)`` after ``normalize(x)``: per element, how far the
    reference's normalised observation may be from this one (float32 batch moments against float64 ones)."""

    def __init__(self, n, d, gamma):
        self.d, self.gamma = d, gamma
        self.obs, self.ret = initial(d), initial(1)
        self.returns = np.zeros(n)
        self.err_mean, self.err_var = np.zeros(d), np.zeros(d)

    def normalize(self, x):
        d, n = self.d, x.shape[0]
        old = self.obs
        self.obs = update(old, moments64(x, old[:d]), d, float(n))
        # float32 np.mean: n - 1 adds and a division, each rounding (Higham, recursive summation); np.var: the
        # deviations from that mean, their squares, n - 1 adds and a division, plus the mean's own error squared
        bm = np.mean(x, axis=0)
        dev = x - bm
        e_bm = gamma_n(n, U32) * np.mean(np.abs(x), axis=0)
        e_bv = gamma_n(n + 3, U32) * np.mean(dev * dev, axis=0) + 2 * e_bm * np.mean(np.abs(dev), axis=0) + e_bm ** 2
        w = n / (old[2 * d] + n)
        delta = np.abs(bm - old[:d])
        e_delta = e_bm + self.err_mean
        self.err_var = (1 - w) * self.err_var + w * e_bv + w * (1 - w) * (2 * delta * e_delta + e_delta ** 2)
        self.err_mean = (1 - w) * self.err_mean + w * e_bm
        return (x - self.obs[:d]) / np.sqrt(self.obs[d:2 * d] + EPS)

    def bound(self, x):
        d = self.d
        sd = np.sqrt(self.obs[d:2 * d] + EPS)
        rel_sd = self.err_var / (2 * (self.obs[d:2 * d] + EPS))
        return (self.err_mean + np.abs(x - self.obs[:d]) * rel_sd) / sd * (1 + 1e-6) + 1e-12 * (1 + np.abs(x) / sd)

    def reward(self, r, done):
        self.returns = self.returns * self.gamma + r
        self.ret = update(self.ret, moments64(self.returns[:, None], self.ret[:1]), 1, float(r.shape[0]))
        out = r / np.sqrt(self.ret[1] + EPS)
        self.returns[done] = 0.0
        return out


def load_fixture(env_id):
    """One id's arrays of tests/golden/reference/normalize_wrappers.npz and the run's parameters."""
    z = np.load(FIXTURE)
    n, t, reset, limit = (int(v) for v in z["events"])
    g = {k.split("/", 1)[1]: z[k] for k in z.files if k.startswith(env_id + "/")}
    return g, dict(n=n, T=t, resets=(0, reset), limit=limit, gamma=float(z["gamma"]), seeds=tuple(z["seeds"]))
