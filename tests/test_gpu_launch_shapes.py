"""The classic-control step at the launch shapes bench.py times, against kernel A bit for bit and against the CPU
oracle under the rules of test_gpu_parity.py.

At these shapes the resident kernels take branches that small batches never reach:
- Kernel B (bulk-copy ring, the CartPole default) refills each of its kBulkStages stages and flips the stage's mbarrier
  parity only when a CTA walks more than kBulkStages tiles.
- The deferred-reset list of a CTA (kBulkResetCap = 512 entries in B, kResetCap = 1024 in P) overflows only when more
  than 46 (B) or 93 (P) sparse warps -- fewer than 12 finishing lanes -- run in one CTA in one launch.  The overflowing
  envs then reset inline.  Whole-batch truncation does not reach it: every warp is dense and resets inline anyway.
- The host path (numpy backend) runs large batches as several chunks on two streams through kernel G, with a ragged
  last chunk and a non-zero first env.
"""
import ctypes
import os

import numpy as np
import pytest

from test_gpu_parity import REW_TOL, _assert_obs

pytestmark = pytest.mark.gpu

ENV_IDS = ["CartPole-v1", "MountainCar-v0", "MountainCarContinuous-v0", "Pendulum-v1", "Acrobot-v1"]
DISCRETE_IDS = ["CartPole-v1", "MountainCar-v0", "Acrobot-v1"]
NTHREADS = os.cpu_count() or 1

# Tiles per SM of the two multi-round shapes (N = tiles * SMs * 256 + 176, a multiple of 16 with a ragged last tile).
# A CTA of B has 288 threads and one of P 256, so an SM holds at most 7 CTAs of B and 8 of P whatever the occupancy:
# at 49 every B CTA walks >= 7 tiles; at 96 every B CTA walks >= 13 and every P CTA >= 12.
SHAPES = {"bulk_shape": 49, "persistent_shape": 96}

# engine variants: kernel A (the reference for the others), B and P
VARIANTS = {
    "a": dict(B200GYM_KERNEL="a"),
    "b": dict(B200GYM_KERNEL="b"),
    "p": dict(B200GYM_KERNEL="p"),
}


def _torch():
    import torch
    return torch


def _shape_n(shape):
    sms = _torch().cuda.get_device_properties(0).multi_processor_count
    return SHAPES[shape] * sms * 256 + 176


def _make(env_id, n, env_vars=None, **kwargs):
    import gym_b200
    with pytest.MonkeyPatch.context() as mp:
        for k in ("B200GYM_KERNEL", "B200GYM_HOST_CHUNKS"):
            mp.delenv(k, raising=False)
        for k, v in (env_vars or {}).items():
            mp.setenv(k, v)
        return gym_b200.vector.make(env_id, n, **kwargs)


def _random_actions(env, gen, dtype=None):
    torch = _torch()
    n = env.num_envs
    if env.discrete:
        return torch.randint(0, env.single_action_space.n, (n,), generator=gen, device=env.device,
                             dtype=dtype or torch.int64)
    lim = 3.0 if env.spec.id.startswith("Pendulum") else 1.5   # beyond the Box bounds: the clip runs too
    return (torch.rand((n, env.act_dim), generator=gen, device=env.device) * 2 - 1) * lim


def _bits(x):
    """A tensor as integers of the same width, so that NaN rewards compare by their bits."""
    torch = _torch()
    if x.dtype == torch.float32:
        return x.view(torch.int32)
    if x.dtype == torch.float64:
        return x.view(torch.int64)
    return x


def _assert_same(ra, rb, what):
    """Every output of one step bit for bit, the final_observation rows under the mask included."""
    torch = _torch()
    for name, x, y in zip(("obs", "reward", "terminated", "truncated"), ra[:4], rb[:4]):
        assert torch.equal(_bits(x), _bits(y)), f"{what}: {name}"
    m = ra[4]["_final_observation"]
    assert torch.equal(m, rb[4]["_final_observation"]), f"{what}: final_observation mask"
    assert torch.equal(_bits(ra[4]["final_observation"][m]), _bits(rb[4]["final_observation"][m])), \
        f"{what}: final_observation rows"


def _assert_same_state(ea, eb, what):
    torch = _torch()
    for name, x, y in zip(("state", "elapsed", "rng"), ea.get_state(), eb.get_state()):
        assert torch.equal(_bits(x), _bits(y)), f"{what}: {name}"


def _check_oracle(env_id, out, ref, what):
    """One step against the oracle (test_gpu_parity.py's rules); returns (bit-identical obs elements, elements)."""
    o, r, te, tr, info = out
    ro, rr, rte, rtr, rfo = ref
    te_h, tr_h = te.cpu().numpy(), tr.cpu().numpy()
    assert np.array_equal(te_h, rte), f"{what}: {np.count_nonzero(te_h != rte)} terminated mismatches"
    assert np.array_equal(tr_h, rtr), f"{what}: {np.count_nonzero(tr_h != rtr)} truncated mismatches"
    o_h = o.cpu().numpy()
    exact = int((o_h == ro).sum())
    if env_id.startswith("CartPole"):
        _assert_obs(o_h, ro, f"{what} obs")
    else:
        assert exact == o_h.size, f"{what}: {o_h.size - exact} observation elements differ from the oracle"
    np.testing.assert_allclose(r.cpu().numpy(), rr, rtol=REW_TOL, atol=REW_TOL, err_msg=what)
    done = rte | rtr
    assert np.array_equal(info["_final_observation"].cpu().numpy(), done), f"{what}: final_observation mask"
    if done.any():
        fo = info["final_observation"].cpu().numpy()[done]
        if env_id.startswith("CartPole"):
            _assert_obs(fo, rfo[done], f"{what} final_observation")
        else:
            assert np.array_equal(fo, rfo[done]), f"{what}: final_observation"
    return exact, o_h.size


def _check_oracle_state(env_id, env, orc, what):
    st, el, rng = env.get_state()
    ost, oel = orc.get_state()
    assert np.array_equal(el.cpu().numpy(), oel), f"{what}: elapsed"
    assert np.array_equal(rng.cpu().numpy().view(np.uint64), orc.get_rng()), f"{what}: rng"
    if env_id.startswith("CartPole"):
        np.testing.assert_allclose(st.cpu().numpy(), ost, rtol=1e-9, atol=1e-9, err_msg=what)
    else:
        assert np.array_equal(st.cpu().numpy(), ost), f"{what}: float64 state"


# ---------------------------------------------------------------------------------------------------------------
# controlled reset density, teacher-forced against the oracle

PATTERNS = ["sparse_11_per_warp", "dense_12_per_warp", "alternating_11_12", "lanes_0_and_31", "ragged_tail_only"]


def _pattern(name, n):
    """Envs that finish in the forced step.  Warps are 32 consecutive envs from env 0 in every kernel."""
    j = np.arange(n)
    lane, warp = j % 32, j // 32
    sparse = lane % 3 == 0          # lanes 0, 3, ..., 30: 11 a warp, one short of the inline threshold
    dense = lane % 8 < 3            # 12 a warp: the inline threshold
    if name == "sparse_11_per_warp":
        return sparse
    if name == "dense_12_per_warp":
        return dense
    if name == "alternating_11_12":
        return np.where(warp % 2 == 0, sparse, dense)
    if name == "lanes_0_and_31":
        return (lane == 0) | (lane == 31)
    assert name == "ragged_tail_only"
    return sparse & (j >= n - n % 256)


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("pattern", PATTERNS)
@pytest.mark.parametrize("env_id", ENV_IDS)
def test_reset_density_teacher_forced(oracle_mod, env_id, pattern, shape):
    """After 3 random steps from reset (no env can finish that early), the pattern's envs get elapsed =
    max_episode_steps - 1 and the same words are loaded into every kernel variant and the oracle; the next step
    truncates exactly the pattern.  11 sparse lanes in every warp put more envs on each CTA's deferred list than it
    holds, in kernel B at both shapes and in kernel P at the persistent shape, so the overflowing envs reset inline;
    12 lanes reset inline from the start.  For CartPole the pattern's envs in even warps also get a pole angle past
    12 degrees, so terminated and truncated coincide there.  Two free steps follow."""
    torch = _torch()
    n = _shape_n(shape)
    envs = {k: _make(env_id, n, v) for k, v in VARIANTS.items()}
    ea = envs["a"]
    for e in envs.values():
        e.reset(seed=5)
    gen = torch.Generator(device=ea.device).manual_seed(17)
    for _ in range(3):
        ea.step(_random_actions(ea, gen))
    st, el, rng = ea.get_state()
    mask_h = _pattern(pattern, n)
    mask = torch.as_tensor(mask_h, device=ea.device)
    el = torch.where(mask, torch.full_like(el, ea.max_episode_steps - 1), el)
    both_h = np.zeros(n, dtype=bool)
    if env_id.startswith("CartPole"):
        both_h = mask_h & ((np.arange(n) // 32) % 2 == 0)
        both = torch.as_tensor(both_h, device=ea.device)
        st[both, 2] = 0.3                # past the 12-degree threshold (0.2094 rad) after one more step
    for e in envs.values():
        e.set_state(state=st, elapsed=el, rng=rng)
    orc = oracle_mod.OracleVec(env_id, n)
    orc.set_state(st.cpu().numpy(), el.cpu().numpy())
    orc.set_rng(rng.cpu().numpy().view(np.uint64))
    exact = total = 0
    for t in range(3):
        a = _random_actions(ea, gen)
        ra = ea.step(a)
        for name, e in envs.items():
            if name != "a":
                _assert_same(ra, e.step(a), f"kernel {name} step {t}")
        x, y = _check_oracle(env_id, ra, orc.step(a.cpu().numpy(), nthreads=NTHREADS), f"oracle step {t}")
        exact, total = exact + x, total + y
        if t == 0:
            assert np.array_equal(ra[3].cpu().numpy(), mask_h), "the forced step truncates exactly the pattern"
            assert np.array_equal(ra[2].cpu().numpy(), both_h), "... and terminates only where the pole was tipped"
    if env_id.startswith("CartPole"):
        assert exact / total > 0.999, f"only {exact / total:.5f} of the observations are bit-identical"
    for name, e in envs.items():
        if name != "a":
            _assert_same_state(ea, e, f"kernel {name}")
    _check_oracle_state(env_id, ea, orc, "oracle")
    for e in envs.values():
        e.close()
    orc.close()


def _invalid_count(env):
    count = ctypes.c_int64(0)
    from gym_b200 import _lib
    _lib.check(env._lib.b200gym_invalid_actions(env._handle, env._stream(), ctypes.byref(count)), env._handle)
    return int(count.value)


@pytest.mark.parametrize("dtype", ["int64", "uint8"])
@pytest.mark.parametrize("env_id", DISCRETE_IDS)
def test_invalid_actions_in_later_round_tiles(env_id, dtype):
    """Out-of-range actions in tiles that resident CTAs reach only in later rounds, and one in the ragged tail: those
    envs keep their state, elapsed and rng, return their current observation and a NaN reward, and each is counted
    once.  Against kernel A only -- the oracle raises on invalid actions, like the reference."""
    torch = _torch()
    n = _shape_n("persistent_shape")
    envs = {k: _make(env_id, n, v) for k, v in VARIANTS.items()}
    ea = envs["a"]
    tdt = getattr(torch, dtype)
    gen = torch.Generator(device=ea.device).manual_seed(3)
    for e in envs.values():
        e.reset(seed=21)
    for _ in range(2):
        a = _random_actions(ea, gen, tdt)
        ra = ea.step(a)
        for name, e in envs.items():
            if name != "a":
                _assert_same(ra, e.step(a), f"kernel {name} warm-up")
    prev_obs = ra[0].clone()
    before = [x.clone() for x in ea.get_state()]
    tiles = n // 256
    rows = torch.tensor([(tiles // 2) * 256 + 3, (tiles // 2) * 256 + 17, (tiles - 2) * 256 + 31, n - 5],
                        device=ea.device)
    nact = ea.single_action_space.n
    bad = [nact, 255, nact + 7, 200] if dtype == "uint8" else [nact, -1, 1 << 40, -(1 << 33)]
    a = _random_actions(ea, gen, tdt)
    a[rows] = torch.tensor(bad, device=ea.device, dtype=tdt)
    outs = {name: e.step(a) for name, e in envs.items()}
    for name, e in envs.items():
        o, r, te, tr, _ = outs[name]
        assert bool(torch.isnan(r[rows]).all()), f"kernel {name}: NaN reward for an invalid action"
        assert int(torch.isnan(r).sum()) == len(bad), f"kernel {name}: NaN only for the invalid actions"
        assert torch.equal(o[rows], prev_obs[rows]), f"kernel {name}: current observation"
        assert not bool(te[rows].any() or tr[rows].any()), f"kernel {name}: flags"
        after = e.get_state()
        for k in range(3):
            assert torch.equal(after[k][rows], before[k][rows]), f"kernel {name}: env left untouched"
        assert _invalid_count(e) == len(bad), f"kernel {name}: invalid-action count"
        if name != "a":
            _assert_same(outs["a"], outs[name], f"kernel {name}")
            _assert_same_state(ea, e, f"kernel {name}")
    for e in envs.values():
        e.close()


# ---------------------------------------------------------------------------------------------------------------
# bench.py's own configurations against the oracle, full batch

# (env_id, N, max_episode_steps, action dtype, steps).  CartPole at 2^20 runs kernel B; at max_episode_steps=37 every
# env that survives 37 steps truncates, at step 37 all at once and from then on in nearly every step, over three
# cycles.  The other kinds at 2^18 run kernel P and run past their TimeLimit once.
BENCH_CASES = [
    pytest.param("CartPole-v1", 1 << 20, None, "int64", 64, id="CartPole-2^20-int64"),
    pytest.param("CartPole-v1", 1 << 20, None, "uint8", 64, id="CartPole-2^20-uint8"),
    pytest.param("CartPole-v1", 1 << 20, 37, "int64", 120, id="CartPole-2^20-int64-limit37"),
    pytest.param("CartPole-v1", 1 << 20, 37, "uint8", 120, id="CartPole-2^20-uint8-limit37"),
    pytest.param("Pendulum-v1", 1 << 18, None, "float32", 210, id="Pendulum-2^18"),
    pytest.param("MountainCar-v0", 1 << 18, None, "int64", 210, id="MountainCar-2^18"),
    pytest.param("Acrobot-v1", 1 << 18, None, "int64", 510, id="Acrobot-2^18"),
]


@pytest.mark.parametrize("env_id,n,max_steps,dtype,steps", BENCH_CASES)
def test_bench_configuration_full_batch(oracle_mod, env_id, n, max_steps, dtype, steps):
    """The default kernel from reset(seed=0) with random actions, every row against the oracle on every step."""
    torch = _torch()
    env = _make(env_id, n, max_episode_steps=max_steps)
    orc = oracle_mod.OracleVec(env_id, n, max_episode_steps=max_steps)
    obs, _ = env.reset(seed=0)
    _assert_obs(obs.cpu().numpy(), orc.reset(seed=0), "reset obs")
    gen = torch.Generator(device=env.device).manual_seed(1)
    tdt = None if dtype == "float32" else getattr(torch, dtype)
    exact = total = n_trunc = trunc_steps = 0
    for t in range(steps):
        a = _random_actions(env, gen, tdt)
        out = env.step(a)
        ref = orc.step(a.cpu().numpy(), nthreads=NTHREADS)
        x, y = _check_oracle(env_id, out, ref, f"step {t}")
        exact, total = exact + x, total + y
        n_trunc += int(ref[3].sum())
        trunc_steps += int(ref[3].any())
    if env_id.startswith("CartPole"):
        assert exact / total > 0.999, f"only {exact / total:.5f} of the observations are bit-identical"
    if max_steps == 37:
        assert trunc_steps >= steps - 2 * max_steps, "truncations in most steps from the first cycle on"
    if not env_id.startswith("CartPole"):
        assert n_trunc >= n // 2
    _check_oracle_state(env_id, env, orc, "final state")
    env.close()
    orc.close()


def test_cartpole_2_23_strong_scaling_line(oracle_mod):
    """2^23 CartPole, bench.py's strong-scaling line on one GPU: a resident CTA walks ~62 tiles and lists ~700
    finishing envs a step.  The default kernel against kernel A bit for bit for 60 steps, and three windows of
    65 536 envs (first, middle, last) against the oracle, each seeded as that slice of the batch."""
    torch = _torch()
    n, T, w = 1 << 23, 60, 1 << 16
    env = _make("CartPole-v1", n)
    ref_env = _make("CartPole-v1", n, VARIANTS["a"])
    windows = [0, n // 2, n - w]
    orcs = []
    for lo in windows:
        orc = oracle_mod.OracleVec("CartPole-v1", w)
        orc.seed(0, first=lo)
        orcs.append(orc)
    obs, _ = env.reset(seed=0)
    assert torch.equal(obs, ref_env.reset(seed=0)[0])
    for lo, orc in zip(windows, orcs):
        assert np.array_equal(obs[lo:lo + w].cpu().numpy(), orc.reset())
    gen = torch.Generator(device=env.device).manual_seed(2)
    exact = total = n_done = 0
    for t in range(T):
        a = _random_actions(env, gen)
        out = env.step(a)
        _assert_same(out, ref_env.step(a), f"default kernel step {t}")
        n_done += int(out[4]["_final_observation"].sum())
        a_h = a.cpu().numpy()
        for lo, orc in zip(windows, orcs):
            sl = slice(lo, lo + w)
            part = (out[0][sl], out[1][sl], out[2][sl], out[3][sl],
                    {"_final_observation": out[4]["_final_observation"][sl],
                     "final_observation": out[4]["final_observation"][sl]})
            x, y = _check_oracle("CartPole-v1", part, orc.step(a_h[sl], nthreads=NTHREADS), f"window {lo} step {t}")
            exact, total = exact + x, total + y
    assert n_done > n
    assert exact / total > 0.999, f"only {exact / total:.5f} of the observations are bit-identical"
    _assert_same_state(env, ref_env, "default kernel")
    st, el, rng = env.get_state()
    for lo, orc in zip(windows, orcs):
        ost, oel = orc.get_state()
        assert np.array_equal(el[lo:lo + w].cpu().numpy(), oel)
        assert np.array_equal(rng[lo:lo + w].cpu().numpy().view(np.uint64), orc.get_rng())
        np.testing.assert_allclose(st[lo:lo + w].cpu().numpy(), ost, rtol=1e-9, atol=1e-9)
        orc.close()
    env.close()
    ref_env.close()


# ---------------------------------------------------------------------------------------------------------------
# the host path (numpy backend) at bench.py's end-to-end shape

# (env_id, N, B200GYM_HOST_CHUNKS or None for the default, steps).  The default splits 2^20 envs into 4 chunks on two
# streams; N = 2^20 + 176 gives every chunk count a ragged last chunk (kernel G's full tiles, kernel A's tail).
HOST_CASES = [
    pytest.param("CartPole-v1", 1 << 20, None, 60, id="CartPole-2^20-default_chunks"),
    pytest.param("CartPole-v1", (1 << 20) + 176, "2", 40, id="CartPole-ragged-2_chunks"),
    pytest.param("CartPole-v1", (1 << 20) + 176, "3", 40, id="CartPole-ragged-3_chunks"),
    pytest.param("CartPole-v1", (1 << 20) + 176, "7", 40, id="CartPole-ragged-7_chunks"),
    pytest.param("Pendulum-v1", 1 << 18, None, 210, id="Pendulum-2^18"),
]


def _assert_host_same(ra, rb, what):
    """torch-backend step ra against numpy-backend step rb (copy=False, dense_infos=True), bit for bit."""
    o, r, te, tr, info = ra
    ho, hr, hte, htr, hinfo = rb
    assert np.array_equal(o.cpu().numpy().view(np.int32), ho.view(np.int32)), f"{what}: obs"
    assert np.array_equal(r.cpu().numpy().view(np.int64), hr.view(np.int64)), f"{what}: reward"
    assert np.array_equal(te.cpu().numpy(), hte) and np.array_equal(tr.cpu().numpy(), htr), f"{what}: flags"
    m = info["_final_observation"].cpu().numpy()
    assert np.array_equal(hinfo["_final_observation"], m), f"{what}: final_observation mask"
    assert np.array_equal(info["final_observation"].cpu().numpy()[m].view(np.int32),
                          hinfo["final_observation"][m].view(np.int32)), f"{what}: final_observation rows"
    return m


@pytest.mark.parametrize("env_id,n,chunks,steps", HOST_CASES)
def test_host_path_chunks(oracle_mod, env_id, n, chunks, steps, monkeypatch):
    """backend="numpy" with copy=False and dense_infos=True (bench.py's end-to-end line) against the torch backend,
    bit for bit with the dense final observations; CartPole at 2^20 also against the oracle."""
    torch = _torch()
    dev = _make(env_id, n)
    host = _make(env_id, n, backend="numpy", copy=False, dense_infos=True)
    if chunks is not None:
        monkeypatch.setenv("B200GYM_HOST_CHUNKS", chunks)   # read at every host step
    with_oracle = n == 1 << 20
    orc = oracle_mod.OracleVec(env_id, n) if with_oracle else None
    o, _ = dev.reset(seed=0)
    ho, _ = host.reset(seed=0)
    assert np.array_equal(o.cpu().numpy(), ho)
    if orc is not None:
        assert np.array_equal(ho, orc.reset(seed=0))
    gen = torch.Generator(device=dev.device).manual_seed(4)
    n_done = 0
    for t in range(steps):
        a = _random_actions(dev, gen)
        a_h = a.cpu().numpy()
        ra = dev.step(a)
        rb = host.step(a_h)
        n_done += int(_assert_host_same(ra, rb, f"step {t}").sum())
        if orc is not None:
            _check_oracle(env_id, ra, orc.step(a_h, nthreads=NTHREADS), f"oracle step {t}")
    assert n_done > 0
    _assert_same_state(dev, host, "host path")
    if orc is not None:
        _check_oracle_state(env_id, dev, orc, "oracle")
        orc.close()
    dev.close()
    host.close()


def test_host_path_invalid_action_in_last_chunk():
    """One out-of-range action in a full tile of the last of 4 chunks (a non-zero first env, stream 1): counted
    exactly once, that env left untouched with a NaN reward, every other env stepped as on the torch backend."""
    import gym_b200
    torch = _torch()
    n = (1 << 20) + 176
    dev = _make("CartPole-v1", n)
    host = _make("CartPole-v1", n, backend="numpy", copy=False, dense_infos=True)
    dev.reset(seed=9)
    host.reset(seed=9)
    gen = torch.Generator(device=dev.device).manual_seed(5)
    for t in range(3):
        a = _random_actions(dev, gen)
        _assert_host_same(dev.step(a), host.step(a.cpu().numpy()), f"step {t}")
    row = n - 176 - 1000           # the last chunk starts at env 787 200 and ends in the ragged tail
    before = [x[row].clone() for x in host.get_state()]
    prev_obs = host._hio["obs"][row].copy()
    a = _random_actions(dev, gen)
    a[row] = 2
    ra = dev.step(a)
    with pytest.raises(gym_b200.error.InvalidAction, match=r"^1 out-of-range"):
        host.step(a.cpu().numpy())
    # the step has run; its results are in the staging buffers that step() would have returned
    h = host._hio
    te, tr = h["terminated"].view(np.bool_), h["truncated"].view(np.bool_)
    rb = (h["obs"], h["reward"], te, tr, {"_final_observation": te | tr, "final_observation": h["final_obs"]})
    _assert_host_same(ra, rb, "invalid step")
    assert np.isnan(rb[1][row]) and int(np.isnan(rb[1]).sum()) == 1
    assert np.array_equal(rb[0][row], prev_obs)
    assert all(torch.equal(x[row], y) for x, y in zip(host.get_state(), before))
    assert _invalid_count(dev) == 1
    _assert_same_state(dev, host, "after the invalid step")
    a = _random_actions(dev, gen)
    _assert_host_same(dev.step(a), host.step(a.cpu().numpy()), "next step")
    dev.close()
    host.close()
