"""The batch normalisers' kernels (``rms_moments_kernel`` / ``rms_apply_kernel``) against exact moments, and the
vector ``NormalizeObservation`` / ``NormalizeReward`` against a float64 restatement at every kind's width.

Kernel level: the four entry points are driven directly on chosen data -- every accepted width, float32 and float64
input, batch sizes around one CTA, around the grid cap (where the grid-stride loop starts to repeat) and at bench
scale.  The batch sums must lie within the worst-case bound of a float64 sum in any order of the exact sum of the
same terms; the Chan update and the normalised outputs are IEEE arithmetic without contraction and must equal a
numpy restatement bit for bit; and the sums must be reproducible bit for bit.
"""
import math
import os
import socket

import numpy as np
import pytest

import normalize_restated as nr

pytestmark = pytest.mark.gpu

WIDTHS = (1, 2, 3, 4, 6, 8, 24)
U = 2.0 ** -53           # unit roundoff of float64
EPS = nr.EPS


def _torch():
    import torch
    return torch


def _lib():
    from gym_b200 import _lib
    return _lib, _lib.load()


def _p(t):
    import ctypes
    return ctypes.c_void_p(t.data_ptr())


def _block(d):
    return 192 if d in (3, 6, 24) else 256


def _grid(total, block):
    return max(1, min(1056, -(-total // block)))


def _rows(d):
    """1, 2; one CTA's worth of rows and one either side; the grid cap and one either side; a ragged bench size."""
    b, cap = _block(d) // d, 1056 * _block(d) // d
    big = 2 ** 21 + 5 if d == 24 else 2 ** 20 + 7
    return sorted({1, 2, b - 1, b, b + 1, cap - 1, cap, cap + 1, big} - {0})


def _columns(d):
    """Per column its own offset and scale: column 0 near 1e4 with a small spread, column 1 constant, the others
    alternating in sign and growing, so that a swapped or shifted column fails."""
    off = np.array([1e4 + 0.37 if c == 0 else 2.5 if c == 1 else (-1) ** c * (c + 1) * 1.7 for c in range(d)])
    scale = np.array([0.01 if c == 0 else 0.0 if c == 1 else 0.1 * (c + 1) for c in range(d)])
    return off, scale


def _data(n, d, dtype, seed):
    off, scale = _columns(d)
    rng = np.random.default_rng(seed)
    return (off + scale * rng.standard_normal((n, d))).astype(dtype)


def _stats(d):
    """A current statistics set with a non-zero pivot (mean) that is not the batch mean, var != 1, count != eps."""
    off, scale = _columns(d)
    mean = off + 0.3 * scale + 0.125
    var = 0.5 + 0.1 * np.arange(d)
    return np.concatenate([mean, var, [137.0]])


def _exact_sum(t):
    """Sum of float64 terms to within a rounding far below the kernel's bound (80-bit long double, or fsum)."""
    if np.finfo(np.longdouble).nmant >= 63:
        return float(np.sum(t.astype(np.longdouble))), t.size.bit_length() * 2.0 ** -63
    return math.fsum(t), 0.0


def _check_moments(xh, d, pivot, got, n_partial_adds=1):
    """got = [sum(x - p), sum((x - p)^2)] per column within (k - 1) u sum|terms| of the exact sums of the kernel's
    terms (float64 x - p and its square are the same IEEE operations in numpy); k = the most additions any term
    can go through: per-thread terms + the CTA's threads of a column + the CTAs (+ the add into scratch)."""
    n = xh.shape[0]
    block = _block(d)
    grid = _grid(n * d, block)
    k = -(-n * d // (grid * block)) + block // d + grid + n_partial_adds
    for c in range(d):
        t = xh[:, c].astype(np.float64) - pivot[c]
        for j, terms in enumerate((t, t * t)):
            want, rel = _exact_sum(terms)
            mag = float(np.sum(np.abs(terms)))
            bound = (k - 1) * U * mag + rel * mag
            err = abs(float(got[j * d + c]) - want)
            assert err <= bound, (n, d, c, "sum" if j == 0 else "sumsq", got[j * d + c], want, err, bound)


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint64 if a.dtype == np.float64 else np.uint32)


def _nan(torch, shape, dtype):
    return torch.full(shape, float("nan"), dtype=dtype, device="cuda")


@pytest.mark.parametrize("is_f64", [0, 1], ids=["f32", "f64"])
@pytest.mark.parametrize("d", WIDTHS)
def test_moments_and_apply_against_exact_sums(d, is_f64):
    torch = _torch()
    _l, lib = _lib()
    st_h = _stats(d)
    stats = torch.as_tensor(st_h, device="cuda")
    work = torch.zeros(_l.rms_work_size(d), dtype=torch.float64, device="cuda")
    for i, n in enumerate(_rows(d)):
        xh = _data(n, d, np.float64 if is_f64 else np.float32, seed=100 * d + i)
        x = torch.as_tensor(xh, device="cuda")
        scratch = torch.zeros(2 * d, dtype=torch.float64, device="cuda")
        _l.check(lib.b200gym_rms_moments(_p(x), is_f64, n, d, _p(stats), _p(scratch), _p(work), None))
        sc = scratch.cpu().numpy()
        _check_moments(xh, d, st_h, sc)
        assert work[0].item() == 0.0, "the CTA ticket must be left at zero for the next launch"
        if is_f64:
            continue
        # apply: the Chan update restated on the device's own sums, bit for bit; a world of two (batch_count 2n)
        for bn, update in ((float(n), 1), (2.0 * n, 1), (float(n), 0)):
            out = _nan(torch, (n, d), torch.float32)
            nxt, nsc = _nan(torch, (2 * d + 1,), torch.float64), _nan(torch, (2 * d,), torch.float64)
            _l.check(lib.b200gym_rms_apply_obs(_p(x), _p(out), n, d, _p(stats), _p(nxt), _p(scratch), _p(nsc), bn, EPS,
                                               update, None))
            if update:
                mean, var, count = nr.chan(st_h, sc, d, bn)
                want = np.concatenate([mean, var, [count]])
                assert np.array_equal(_bits(nxt.cpu().numpy()), _bits(want)), (n, d, bn)
                assert np.array_equal(_bits(nsc.cpu().numpy()), np.zeros(2 * d, np.uint64)), "scratch_next not zeroed"
            else:
                mean, var = st_h[:d], st_h[d:2 * d]
                assert np.isnan(nxt.cpu().numpy()).all() and np.isnan(nsc.cpu().numpy()).all(), "update=0 wrote"
            ref = ((xh.astype(np.float64) - mean) / np.sqrt(var + EPS)).astype(np.float32)
            got = out.cpu().numpy()
            assert np.array_equal(_bits(got), _bits(ref)), (n, d, bn, update, int((_bits(got) != _bits(ref)).sum()))


def test_return_moments_and_apply_reward():
    torch = _torch()
    _l, lib = _lib()
    st_h = np.array([0.75, 2.5, 41.0])
    stats = torch.as_tensor(st_h, device="cuda")
    work = torch.zeros(_l.rms_work_size(1), dtype=torch.float64, device="cuda")
    gamma = 0.9
    for i, n in enumerate(_rows(1)):
        rng = np.random.default_rng(7 + i)
        ret_h = rng.standard_normal(n) * 3.0 + 1.0
        rew_h = rng.standard_normal(n) * 0.5 - 0.2
        # every flag combination: none, terminated alone, truncated alone, both
        term_h = (np.arange(n) % 4 == 1) | (np.arange(n) % 4 == 3)
        trunc_h = (np.arange(n) % 4 == 2) | (np.arange(n) % 4 == 3)
        returns, reward = torch.as_tensor(ret_h, device="cuda"), torch.as_tensor(rew_h, device="cuda")
        term = torch.as_tensor(term_h.astype(np.uint8), device="cuda")
        trunc = torch.as_tensor(trunc_h.astype(np.uint8), device="cuda")
        scratch = torch.zeros(2, dtype=torch.float64, device="cuda")
        _l.check(lib.b200gym_return_moments(_p(returns), _p(reward), gamma, n, _p(stats), _p(scratch), _p(work), None))
        new_ret = ret_h * gamma + rew_h                                            # normalize.py:130, no contraction
        assert np.array_equal(_bits(returns.cpu().numpy()), _bits(new_ret)), n
        sc = scratch.cpu().numpy()
        _check_moments(new_ret[:, None], 1, st_h, sc)
        out = _nan(torch, (n,), torch.float64)
        nxt, nsc = _nan(torch, (3,), torch.float64), _nan(torch, (2,), torch.float64)
        _l.check(lib.b200gym_rms_apply_reward(_p(reward), _p(out), _p(returns), _p(term), _p(trunc), n, _p(stats),
                                              _p(nxt), _p(scratch), _p(nsc), 2.0 * n, EPS, None))
        mean, var, count = nr.chan(st_h, sc, 1, 2.0 * n)
        assert np.array_equal(_bits(nxt.cpu().numpy()), _bits(np.concatenate([mean, var, [count]]))), n
        assert np.array_equal(_bits(nsc.cpu().numpy()), np.zeros(2, np.uint64))
        assert np.array_equal(_bits(out.cpu().numpy()), _bits(rew_h / np.sqrt(var + EPS))), n
        want_ret = np.where(term_h | trunc_h, 0.0, new_ret)                        # :135-136
        assert np.array_equal(_bits(returns.cpu().numpy()), _bits(want_ret)), n


@pytest.mark.parametrize("d", (5, 7, 16, 25))
def test_unsupported_widths_are_refused_without_a_launch(d):
    torch = _torch()
    _l, lib = _lib()
    n = 1000
    x = torch.ones((n, d), dtype=torch.float32, device="cuda")
    stats = torch.zeros(2 * d + 1, dtype=torch.float64, device="cuda")
    scratch = _nan(torch, (2 * d,), torch.float64)
    work = torch.zeros(_l.rms_work_size(max(d, 1)), dtype=torch.float64, device="cuda")
    assert lib.b200gym_rms_moments(_p(x), 0, n, d, _p(stats), _p(scratch), _p(work), None) != 0
    assert "dim must be one of 1, 2, 3, 4, 6, 8, 24" in _l.last_error()
    out = _nan(torch, (n, d), torch.float32)
    nxt, nsc = _nan(torch, (2 * d + 1,), torch.float64), _nan(torch, (2 * d,), torch.float64)
    assert lib.b200gym_rms_apply_obs(_p(x), _p(out), n, d, _p(stats), _p(nxt), _p(scratch), _p(nsc), float(n), EPS, 1,
                                     None) != 0
    assert "dim must be one of 1, 2, 3, 4, 6, 8, 24" in _l.last_error()
    torch.cuda.synchronize()
    for t in (scratch, out, nxt, nsc):
        assert torch.isnan(t).all(), "a refused call launched"
    assert not work.any()


@pytest.mark.parametrize("d", (1, 3, 24))
def test_moments_are_reproducible_bit_for_bit(d):
    """The same inputs into fresh scratch give the same sums, bit for bit (2^20 rows: the grid-stride loop runs)."""
    torch = _torch()
    _l, lib = _lib()
    n = 2 ** 20
    gen = torch.Generator(device="cuda").manual_seed(d)
    off, scale = (torch.as_tensor(a, device="cuda") for a in _columns(d))
    x = (off + scale * torch.randn((n, d), generator=gen, dtype=torch.float64, device="cuda")).float()
    stats = torch.as_tensor(_stats(d), device="cuda")
    runs = []
    for _ in range(2):
        scratch = torch.zeros(2 * d, dtype=torch.float64, device="cuda")
        work = torch.zeros(_l.rms_work_size(d), dtype=torch.float64, device="cuda")
        _l.check(lib.b200gym_rms_moments(_p(x), 0, n, d, _p(stats), _p(scratch), _p(work), None))
        runs.append(scratch.cpu().numpy())
    assert np.array_equal(_bits(runs[0]), _bits(runs[1])), runs


# ---- the vector wrappers at every kind's width ---------------------------------------------------------------------
def _close_stats(got, want, d, what):
    """{mean, var, count} to 1e-12: a mean relative to its magnitude plus the standard deviation (a mean near zero
    carries the rounding of sums of order n * sd), the variance and the count relative to themselves."""
    sd = np.sqrt(want[d:2 * d])
    err = np.concatenate([np.abs(got[:d] - want[:d]) / (np.abs(want[:d]) + sd),
                          np.abs(got[d:] - want[d:]) / np.abs(want[d:])])
    assert float(err.max()) <= 1e-12, (what, float(err.max()), int(err.argmax()))


def _ulp_ok(got, want64, what):
    want = want64.astype(np.float32)
    gi, wi = got.astype(np.float32).view(np.int32).astype(np.int64), want.view(np.int32).astype(np.int64)
    diff = np.abs(gi - wi)
    assert int(diff.max()) <= 1, (what, int(diff.max()))
    assert float((diff == 0).mean()) >= 0.999, (what, float((diff == 0).mean()))


def _actions(env, rng, n):
    if env.discrete:
        return rng.integers(0, env.single_action_space.n, size=n)
    return rng.uniform(-1.5, 1.5, size=(n, env.act_dim)).astype(np.float32)


WRAPPER_CASES = [("CartPole-v1", 2 ** 20, 11, None), ("MountainCar-v0", 2 ** 18, 9, None),
                 ("MountainCarContinuous-v0", 2 ** 18, 9, None), ("Pendulum-v1", 2 ** 18, 9, None),
                 ("Acrobot-v1", 2 ** 18, 9, None), ("LunarLander-v2", 2 ** 16, 9, None),
                 ("BipedalWalker-v3", 2 ** 16, 9, None), ("CartPole-v1", 2 ** 18, 11, 6)]


@pytest.mark.parametrize("env_id,n,limit,stack", WRAPPER_CASES,
                         ids=[f"{e}-{n}" + (f"-stack{s}" if s else "") for e, n, _, s in WRAPPER_CASES])
def test_wrappers_against_a_float64_restatement(env_id, n, limit, stack):
    import gym_b200
    from gym_b200 import subenv
    from gym_b200.wrappers import NormalizeObservation, NormalizeReward
    kw = dict(max_episode_steps=limit)
    if stack:
        kw["wrappers"] = [subenv.FrameStack(stack)]
    env = NormalizeReward(NormalizeObservation(gym_b200.vector.make(env_id, n, **kw)), gamma=0.9)
    twin = gym_b200.vector.make(env_id, n, **kw)
    d = env.env.obs_rms.d
    ref = nr.Restated64(n, d, 0.9)
    rng = np.random.default_rng(1)
    T, n_done = 24, 0
    for t in range(T + 1):
        if t in (0, 13):                                              # reset, and a mid-run reset(seed=)
            o, _ = env.reset(seed=40 + t)
            raw, _ = twin.reset(seed=40 + t)
            x = raw.cpu().numpy().reshape(n, d).astype(np.float64)
            _ulp_ok(o.cpu().numpy().reshape(n, d), ref.normalize(x), (env_id, "reset", t))
            continue
        a = _actions(twin, rng, n)
        o, r, te, tr, _ = env.step(a)
        raw, rr, rte, rtr, _ = twin.step(a)
        assert np.array_equal(te.cpu().numpy(), rte.cpu().numpy()) and np.array_equal(tr.cpu().numpy(), rtr.cpu().numpy())
        x = raw.cpu().numpy().reshape(n, d).astype(np.float64)
        _ulp_ok(o.cpu().numpy().reshape(n, d), ref.normalize(x), (env_id, "obs", t))
        done = (rte | rtr).cpu().numpy()
        n_done += int(done.sum())
        want_r = ref.reward(rr.cpu().numpy(), done)
        np.testing.assert_allclose(r.cpu().numpy(), want_r, rtol=1e-12, atol=0, err_msg=f"{env_id} reward {t}")
        for rms, want in ((env.env.obs_rms, ref.obs), (env.return_rms, ref.ret)):
            _close_stats(rms.stats[rms.cur].cpu().numpy(), want, rms.d, (env_id, "statistics", t))
        np.testing.assert_allclose(env.returns.cpu().numpy(), ref.returns, rtol=1e-12, atol=1e-300)
    assert n_done > 0, "the TimeLimit must have reset some envs"
    env.close()
    twin.close()


def test_unsupported_width_is_refused_at_construction():
    import gym_b200
    from gym_b200 import subenv
    from gym_b200.wrappers import NormalizeObservation
    env = gym_b200.vector.make("CartPole-v1", 64, wrappers=[subenv.FrameStack(4)])   # 4 x 4 = 16 per row
    with pytest.raises(ValueError, match="1, 2, 3, 4, 6, 8, 24"):
        NormalizeObservation(env)
    env.close()


def test_normalised_rollouts_are_deterministic():
    """Two normalised envs, same seed, same actions: every output bit for bit (tests/envs/test_envs.py:60-115 of
    the reference, on the vector normalisers at a size where every moments launch grid-strides)."""
    import gym_b200
    from gym_b200.wrappers import NormalizeObservation, NormalizeReward
    n = 2 ** 19
    envs = [NormalizeReward(NormalizeObservation(gym_b200.vector.make("Acrobot-v1", n, max_episode_steps=20)))
            for _ in range(2)]
    outs = [e.reset(seed=3) for e in envs]
    assert np.array_equal(_bits(outs[0][0].cpu().numpy()), _bits(outs[1][0].cpu().numpy()))
    rng = np.random.default_rng(5)
    for t in range(40):
        a = rng.integers(0, 3, size=n)
        s0, s1 = (e.step(a) for e in envs)
        for u, v in zip(s0[:4], s1[:4]):
            assert np.array_equal(u.cpu().numpy().view(np.uint8), v.cpu().numpy().view(np.uint8)), t
    for k in ("obs_rms", "return_rms"):
        a, b = (getattr(e, k) if k == "return_rms" else getattr(e.env, k) for e in envs)
        assert np.array_equal(_bits(a.stats.cpu().numpy()), _bits(b.stats.cpu().numpy())), k
    for e in envs:
        e.close()


@pytest.mark.parametrize("env_id", ["CartPole-v1", "MountainCar-v0", "MountainCarContinuous-v0", "Pendulum-v1",
                                    "Acrobot-v1"])
def test_wrappers_against_the_reference_fixture(env_id):
    """The engine's normalisers over the seeds and actions frozen from the reference's own wrappers
    (tests/golden/reference/normalize_wrappers.npz): flags exactly, observations within the bound the reference's
    float32 batch moments allow plus the engine's float32 rounding, rewards to 1e-12."""
    import gym_b200
    from gym_b200.wrappers import NormalizeObservation, NormalizeReward
    g, m = nr.load_fixture(env_id)
    n = m["n"]
    env = NormalizeReward(NormalizeObservation(gym_b200.vector.make(env_id, n, max_episode_steps=m["limit"])),
                          gamma=m["gamma"])
    twin = gym_b200.vector.make(env_id, n, max_episode_steps=m["limit"])
    res = nr.Restated64(n, g["raw_obs"].shape[2], m["gamma"])
    for t in range(m["T"]):
        if t in m["resets"]:
            seed = int(m["seeds"][t != 0])
            o, _ = env.reset(seed=seed)
            raw, _ = twin.reset(seed=seed)
        else:
            a = g["actions"][t]
            o, r, te, tr, _ = env.step(a)
            raw, rr, *_ = twin.step(a)
            assert np.array_equal(te.cpu().numpy(), g["terminated"][t]), t
            assert np.array_equal(tr.cpu().numpy(), g["truncated"][t]), t
            # raw rewards as the engine's parity tests allow (Pendulum's float32 torque cost: DESIGN §4, Numerics),
            # scaled exactly as the reference scaled its own
            rr = rr.cpu().numpy()
            np.testing.assert_allclose(rr, g["raw_reward"][t], rtol=1e-9, atol=1e-9, err_msg=str(t))
            np.testing.assert_allclose(r.cpu().numpy(), rr / np.sqrt(g["ret_var"][t] + EPS), rtol=1e-12, atol=0,
                                       err_msg=str(t))
        x_ref = g["raw_obs"][t].astype(np.float64)
        res.normalize(x_ref)
        # the engine's raw rows may differ from the reference's in the last float32 bits (DESIGN §2); such a
        # difference moves the output by at most itself over the standard deviation, for the row and for the mean
        sd = np.sqrt(res.obs[res.d:2 * res.d] + EPS)
        raw_diff = np.abs(raw.cpu().numpy().astype(np.float64) - x_ref).max(axis=0)
        got = o.cpu().numpy().astype(np.float64)
        want = g["obs"][t]
        bound = res.bound(x_ref) + np.spacing(np.abs(want).astype(np.float32)) + 3 * raw_diff / sd * (1 + np.abs(want))
        assert (np.abs(got - want) <= bound).all(), (t, float((np.abs(got - want) / bound).max()))
    env.close()
    twin.close()


# ---- shards of unequal size ----------------------------------------------------------------------------------------
def _ngpus():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


def _unequal_shard_worker(rank, world, port, q):
    """Shards of 2999 and 3001 envs, batch moments all-reduced, against one env of 6000 on one GPU."""
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        import gym_b200
        from gym_b200.wrappers import NormalizeObservation, NormalizeReward
        sizes = (2999, 3001)
        total, lo = sum(sizes), sum(sizes[:rank])
        hi = lo + sizes[rank]
        full = NormalizeReward(NormalizeObservation(gym_b200.vector.make("Pendulum-v1", total, max_episode_steps=13)),
                               gamma=0.9)
        shard = NormalizeReward(NormalizeObservation(
            gym_b200.vector.make("Pendulum-v1", sizes[rank], max_episode_steps=13, first_index=lo), group=True),
            gamma=0.9, group=True)
        fo, _ = full.reset(seed=5)
        so, _ = shard.reset(seed=5)
        torch.testing.assert_close(so, fo[lo:hi], rtol=1e-6, atol=1e-6)
        rng = np.random.default_rng(0)
        for t in range(30):
            a = torch.as_tensor(rng.uniform(-2, 2, size=(total, 1)).astype(np.float32), device="cuda")
            fo, fr, _, _, _ = full.step(a)
            so, sr, _, _, _ = shard.step(a[lo:hi])
            torch.testing.assert_close(so, fo[lo:hi], rtol=1e-6, atol=1e-6)
            torch.testing.assert_close(sr, fr[lo:hi], rtol=1e-10, atol=1e-12)
        for s, f in ((shard.env.obs_rms, full.env.obs_rms), (shard.return_rms, full.return_rms)):
            torch.testing.assert_close(s.stats[s.cur], f.stats[f.cur], rtol=1e-10, atol=1e-12)
        full.close()
        shard.close()
        q.put((rank, "ok"))
    except Exception:  # pragma: no cover
        import traceback
        q.put((rank, traceback.format_exc()))
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(_ngpus() < 2, reason="needs at least 2 GPUs")
@pytest.mark.timeout(300)
def test_unequal_shards_count_their_rows():
    import torch.multiprocessing as mp
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    procs = [ctx.Process(target=_unequal_shard_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = dict(q.get(timeout=240) for _ in range(world))
    for p in procs:
        p.join(timeout=30)
    assert all(v == "ok" for v in results.values()), results
