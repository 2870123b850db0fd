"""Kernel B resets every finishing env inside the tile's shared-memory stage, fetching the PCG64 records of the envs
that CartPole's lookahead predicts before it steps them.  Against kernel A (one tile per CTA, plain loads and stores,
resets after a CTA barrier): every step's outputs and final observations, and at the end the envs' snapshots (state,
TimeLimit counter, PCG64 record, flags), must be bit-identical -- whatever the prediction says, and at the shapes
bench.py times."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ENV_ID = "CartPole-v1"


def _pair(n, monkeypatch, **kw):
    import gym_b200
    envs = []
    for k in ("a", "b"):
        monkeypatch.setenv("B200GYM_KERNEL", k)
        envs.append(gym_b200.vector.make(ENV_ID, n, **kw))
    monkeypatch.delenv("B200GYM_KERNEL")
    return envs


def _bits(x):
    """x with its float elements as integers of the same width: NaN rewards compare bit for bit"""
    import torch
    return x.view({torch.float64: torch.int64, torch.float32: torch.int32}.get(x.dtype, x.dtype))


def _step_both(ea, eb, a, what):
    import torch
    ra, rb = ea.step(a), eb.step(a)
    for name, x, y in zip(("obs", "reward", "terminated", "truncated"), ra[:4], rb[:4]):
        assert torch.equal(_bits(x), _bits(y)), f"{what}: {name}"
    ia, ib = ra[4], rb[4]
    if "_final_observation" in ia:
        m = ia["_final_observation"]
        assert torch.equal(m, ib["_final_observation"]), f"{what}: final-observation mask"
        assert torch.equal(_bits(ia["final_observation"][m]), _bits(ib["final_observation"][m])), \
            f"{what}: final observations"
    return ra


def _assert_same_snapshot(ea, eb):
    import torch
    sa, sb = ea.snapshot(), eb.snapshot()
    assert torch.equal(sa.rows, sb.rows), "snapshot rows (state, counter, PCG64 record, flags)"
    for x, y in zip(ea.get_state(), eb.get_state()):
        assert torch.equal(x, y), "state"


def _actions(n, seed, dtype):
    import torch
    gen = torch.Generator(device="cuda").manual_seed(seed)
    return [torch.randint(0, 2, (n,), device="cuda", generator=gen).to(getattr(torch, dtype)) for _ in range(8)]


# (envs, steps, max_episode_steps, action dtype, autoreset)
CASES = [
    pytest.param(1 << 20, 600, None, "int64", True, id="2^20-600steps-timelimit"),
    pytest.param(1 << 23, 60, None, "int64", True, id="2^23"),
    pytest.param((1 << 20) + 176, 120, None, "int64", True, id="2^20+176-ragged"),
    pytest.param(1 << 20, 8, 1, "int64", True, id="2^20-limit1"),
    pytest.param(1 << 20, 8, 2, "int64", True, id="2^20-limit2"),
    pytest.param(1 << 20, 120, None, "int64", False, id="2^20-no-autoreset"),
    pytest.param(1 << 20, 120, 50, "uint8", True, id="2^20-uint8"),
    pytest.param(1 << 20, 120, 50, "int32", True, id="2^20-int32"),
]


@pytest.mark.parametrize("n,steps,max_steps,dtype,autoreset", CASES)
def test_kernel_b_equals_kernel_a(n, steps, max_steps, dtype, autoreset, monkeypatch):
    import torch
    kw = {"autoreset": autoreset}
    if max_steps is not None:
        kw["max_episode_steps"] = max_steps
    ea, eb = _pair(n, monkeypatch, **kw)
    assert torch.equal(ea.reset(seed=5)[0], eb.reset(seed=5)[0])
    pool = _actions(n, 17, dtype)
    finished = 0
    for t in range(steps):
        r = _step_both(ea, eb, pool[t % len(pool)], f"step {t}")
        finished += int((r[2] | r[3]).sum())
    _assert_same_snapshot(ea, eb)
    assert finished > 0
    if max_steps is not None and max_steps <= 2:
        assert finished >= n * (steps // max_steps)   # every env finishes at least every max_steps steps
    ea.close()
    eb.close()


@pytest.mark.parametrize("dtype", ["int64", "uint8"])
def test_invalid_actions_on_predicted_envs(dtype, monkeypatch):
    """Out-of-range actions on envs whose state says they terminate on this step (the lookahead marks them, and kernel
    B fetches their records): they must be left untouched, with a NaN reward, exactly as kernel A leaves them."""
    import torch
    from gym_b200 import error
    n = 1 << 20
    ea, eb = _pair(n, monkeypatch)
    ea.reset(seed=8)
    eb.reset(seed=8)
    pool = _actions(n, 4, dtype)
    for t in range(30):
        _step_both(ea, eb, pool[t % len(pool)], f"warm-up step {t}")
    s = ea.get_state()[0].cpu().numpy()
    x, theta = s[:, 0] + 0.02 * s[:, 1], s[:, 2] + 0.02 * s[:, 3]   # numpy: no contraction, as the device code
    marked = np.flatnonzero((np.abs(x) > 2.4) | (np.abs(theta) > 12 * 2 * np.pi / 360))
    assert marked.size > 100
    rows = torch.as_tensor(marked[:: max(1, marked.size // 300)], device="cuda")
    a = pool[0].clone()
    bad = [2, 255] if dtype == "uint8" else [2, -1]
    a[rows] = torch.tensor(bad, device="cuda", dtype=a.dtype).repeat(rows.numel())[: rows.numel()]
    before = [x.clone() for x in ea.get_state()]
    r = _step_both(ea, eb, a, "invalid step")
    assert int(torch.isnan(r[1]).sum()) == rows.numel() and bool(torch.isnan(r[1][rows]).all())
    for k, x in enumerate(eb.get_state()):
        assert torch.equal(x[rows], before[k][rows]), "kernel b: env left untouched"
    others = torch.ones(n, dtype=torch.bool, device="cuda")
    others[rows] = False
    assert bool((r[2] | r[3])[others].any()), "the valid envs still finish"
    for e in (ea, eb):
        with pytest.raises(error.InvalidAction):
            e.check_actions()
    for t in range(10):
        _step_both(ea, eb, pool[(t + 1) % len(pool)], f"step {t} after")
    _assert_same_snapshot(ea, eb)
    ea.close()
    eb.close()
