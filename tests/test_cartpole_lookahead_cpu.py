"""Kernel B's CartPole lookahead, in the host build of the device source: `Env<CARTPOLE>::will_terminate` must equal
the `terminated` that `step` computes, and `will_reset` must equal `advance_env`'s "reset this env", bit for bit.
Kernel B only uses the prediction to fetch PCG64 records early, so a mismatch would cost time, not results; these
tests pin that the prediction is exact, including at the thresholds' last ulps and for NaN / inf state words."""
import numpy as np
import pytest

from hostsim import lookahead_sim as sim

TAU, X_THR, THETA_THR = 0.02, 2.4, 12 * 2 * np.pi / 360


def _check(state, elapsed=0, actions=0, max_steps=500, autoreset=True):
    pred_term, step_term, pred_reset, step_reset = sim.cartpole_lookahead(state, elapsed, actions, max_steps, autoreset)
    bad = np.flatnonzero(pred_term != step_term)
    assert bad.size == 0, f"will_terminate differs from step on {bad.size} states, e.g. {state[bad[0]]!r}"
    bad = np.flatnonzero(pred_reset != step_reset)
    assert bad.size == 0, f"will_reset differs from advance_env on {bad.size} states, e.g. {state[bad[0]]!r}"
    return step_term, step_reset


def test_random_states():
    """10^7 states: most where episodes live and end (the next x or theta on either side of its threshold), some
    anywhere in the float64 range"""
    rng = np.random.default_rng(20261017)
    n = 10_000_000
    scale = np.array([3.0, 4.0, 0.5, 4.0])
    s = rng.uniform(-1.0, 1.0, size=(n, 4)) * scale
    wide = rng.random(n) < 0.05
    s[wide] = rng.standard_normal((int(wide.sum()), 4)) * 10.0 ** rng.uniform(-300, 300, size=(int(wide.sum()), 4))
    term, _ = _check(s)
    assert 0.2 < term.mean() < 0.8


@pytest.mark.parametrize("which,thr", [(0, X_THR), (0, -X_THR), (2, THETA_THR), (2, -THETA_THR)])
def test_states_at_the_thresholds(which, thr):
    """the position word (x or theta) placed within 8 ulps of the threshold after the Euler step, with and without
    a velocity in the step"""
    rng = np.random.default_rng([which, int(thr > 0)])
    n = 200_000
    s = rng.uniform(-0.01, 0.01, size=(n, 4))   # the other position word stays far from its threshold
    vel = rng.uniform(-2.0, 2.0, size=n)
    vel[: n // 4] = 0.0
    s[:, which + 1] = vel
    target = np.full(n, thr)
    for _ in range(4):   # walk the start to the state whose step lands on the threshold, then up to 8 ulps off it
        target += thr - (target + TAU * vel)
    steps = rng.integers(-8, 9, size=n)
    pos = target.copy()
    for k in range(8):
        pos = np.where(steps > k, np.nextafter(pos, np.inf), pos)
        pos = np.where(steps < -k, np.nextafter(pos, -np.inf), pos)
    s[:, which] = pos
    term, _ = _check(s)
    nxt = pos + TAU * vel
    assert np.any(nxt == thr) and term.any() and not term.all()


def test_nan_and_inf_components():
    specials = np.array([np.nan, -np.nan, np.inf, -np.inf, 0.0, -0.0, X_THR, -X_THR, THETA_THR, 1e308, -1e308,
                         5e-324])
    grid = np.stack(np.meshgrid(*([specials] * 4), indexing="ij"), axis=-1).reshape(-1, 4)
    _check(grid)


@pytest.mark.parametrize("autoreset", [True, False])
def test_reset_prediction_with_time_limit_and_invalid_actions(autoreset):
    """will_reset folds in TimeLimit truncation, autoreset and the action's range check exactly as advance_env"""
    rng = np.random.default_rng(7)
    n = 400_000
    s = rng.uniform(-1.0, 1.0, size=(n, 4)) * np.array([3.0, 4.0, 0.5, 4.0])
    elapsed = rng.integers(0, 6, size=n).astype(np.int32)
    actions = rng.choice(np.array([0, 1, -1, 2, 255, -(2**63)]), size=n, p=[0.4, 0.4, 0.05, 0.05, 0.05, 0.05])
    for max_steps in (0, 1, 2, 5):
        _, reset = _check(s, elapsed, actions, max_steps, autoreset)
        if autoreset:
            assert reset.any() and not reset.all()
        else:
            assert not reset.any()
