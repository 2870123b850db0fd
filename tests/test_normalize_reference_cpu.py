"""The reference's vector NormalizeReward(NormalizeObservation(SyncVectorEnv)) frozen in
tests/golden/reference/normalize_wrappers.npz (oracle/gen_normalize_fixtures.py), against the restatements in
tests/normalize_restated.py: the reference's own arithmetic bit for bit, and the float64 arithmetic of the device
normalisers within the bound that the reference's float32 batch moments allow."""
import numpy as np
import pytest

import normalize_restated as nr

CLASSIC = ["CartPole-v1", "MountainCar-v0", "MountainCarContinuous-v0", "Pendulum-v1", "Acrobot-v1"]
load = nr.load_fixture


def _bits(a):
    return np.ascontiguousarray(np.asarray(a, np.float64)).view(np.uint64)


@pytest.mark.parametrize("env_id", CLASSIC)
def test_reference_restatement_reproduces_the_fixture_bit_for_bit(env_id):
    g, m = load(env_id)
    ref = nr.Reference(m["n"], g["raw_obs"].shape[2], m["gamma"])
    for t in range(m["T"]):
        o = ref.normalize(g["raw_obs"][t])
        assert np.array_equal(_bits(o), _bits(g["obs"][t])), t
        if t not in m["resets"]:
            r = ref.reward(g["raw_reward"][t], g["terminated"][t] | g["truncated"][t])
            assert np.array_equal(_bits(r), _bits(g["reward"][t])), t
        assert np.array_equal(_bits(ref.returns), _bits(g["returns"][t])), t
        for got, key in ((ref.obs_mean, "obs_mean"), (ref.obs_var, "obs_var"), (ref.obs_count, "obs_count"),
                         (ref.ret_mean, "ret_mean"), (ref.ret_var, "ret_var"), (ref.ret_count, "ret_count")):
            assert np.array_equal(_bits(got), _bits(g[key][t])), (t, key)


@pytest.mark.parametrize("env_id", CLASSIC)
def test_float64_restatement_within_the_float32_moments_bound(env_id):
    """The device normalisers' float64 arithmetic departs from the reference only by the float32 accumulation of
    np.mean / np.var over the batch: every normalised observation within the propagated bound, rewards to 1e-12."""
    g, m = load(env_id)
    n, d = m["n"], g["raw_obs"].shape[2]
    res = nr.Restated64(n, d, m["gamma"])
    worst = 0.0
    for t in range(m["T"]):
        x = g["raw_obs"][t].astype(np.float64)
        o = res.normalize(x)
        b = res.bound(x)
        err = np.abs(o - g["obs"][t])
        assert (err <= b).all(), (t, float((err / b).max()))
        worst = max(worst, float((err / b).max()))
        if t not in m["resets"]:
            r = res.reward(g["raw_reward"][t], g["terminated"][t] | g["truncated"][t])
            np.testing.assert_allclose(r, g["reward"][t], rtol=1e-12, atol=0, err_msg=str(t))
        np.testing.assert_allclose(res.obs[:d], g["obs_mean"][t], rtol=0, atol=float(res.err_mean.max()) * 1.01 + 1e-15)
    assert worst > 0.0   # float32 moments differ from float64 ones somewhere: the bound is exercised
