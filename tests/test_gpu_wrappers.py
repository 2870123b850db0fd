"""Device-side vector wrappers (SURVEY.md 8f) against numpy restatements of the reference wrappers."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _update_moments(mean, var, count, x):
    # gym/wrappers/normalize.py:19-46
    bm, bv, bc = np.mean(x, axis=0), np.var(x, axis=0), x.shape[0]
    delta = bm - mean
    tot = count + bc
    new_mean = mean + delta * bc / tot
    m2 = var * count + bv * bc + np.square(delta) * count * bc / tot
    return new_mean, m2 / tot, tot


def test_record_episode_statistics():
    import gym_b200
    import torch
    from gym_b200.wrappers import RecordEpisodeStatistics
    N, T = 4096, 120
    env = RecordEpisodeStatistics(gym_b200.vector.make("CartPole-v1", N), deque_size=64)
    env.reset(seed=0)
    ret = np.zeros(N, np.float32)
    length = np.zeros(N, np.int32)
    gen = torch.Generator(device="cuda").manual_seed(1)
    finished = []
    for t in range(T):
        a = torch.randint(0, 2, (N,), device="cuda", generator=gen)
        obs, rew, term, trunc, infos = env.step(a)
        r, done = rew.cpu().numpy(), (term | trunc).cpu().numpy()
        ret += r                      # record_episode_statistics.py:116-117 (float32 accumulator)
        length += 1
        assert np.array_equal(infos["_episode"].cpu().numpy(), done)
        assert np.array_equal(infos["episode"]["r"].cpu().numpy()[done], ret[done])
        assert np.array_equal(infos["episode"]["l"].cpu().numpy()[done], length[done])
        assert infos["episode"]["r"].dtype == torch.float32 and infos["episode"]["l"].dtype == torch.int32
        assert "final_observation" in infos and isinstance(infos["episode"]["t"], float)
        finished += list(zip(ret[done].tolist(), length[done].tolist()))
        ret[done] = 0
        length[done] = 0
    assert env.episode_count == len(finished) > N
    rq, lq = env.return_queue, env.length_queue
    assert len(rq) == 64 and len(lq) == 64
    # CartPole returns equal lengths (reward 1 per step); every ring slot holds ONE finished episode even though
    # ~190 episodes finish per step here and several of them land on the same slot (64-bit packed store)
    assert all(float(a) == float(b) for a, b in zip(rq, lq))
    assert set(zip(rq, lq)) <= set(finished)
    env.close()


def test_episode_statistics_equal_a_numpy_restatement():
    """Every step's accumulators, episode rows, `_episode` mask and episode count against
    record_episode_statistics.py:116-139 restated in numpy over the rewards and flags step() returned, for a
    classic-control kind, float rewards with a short TimeLimit and a Box2D kind."""
    import gym_b200
    import torch
    from gym_b200.wrappers import RecordEpisodeStatistics
    for env_id, N, T, kw in (("CartPole-v1", 3000, 80, {}), ("Pendulum-v1", 1500, 60, dict(max_episode_steps=17)),
                             ("LunarLander-v2", 512, 140, {})):
        env = RecordEpisodeStatistics(gym_b200.vector.make(env_id, N, **kw), deque_size=0)
        env.reset(seed=21)
        ret = np.zeros(N, np.float32)
        length = np.zeros(N, np.int32)
        count = 0
        gen = torch.Generator(device="cuda").manual_seed(3)
        inner = env.env
        for t in range(T):
            if inner.discrete:
                a = torch.randint(0, inner.single_action_space.n, (N,), device="cuda", generator=gen)
            else:
                a = torch.rand((N, inner.act_dim), device="cuda", generator=gen) * 4 - 2
            _, rew, term, trunc, infos = env.step(a)
            r = rew.cpu().numpy()
            assert r.dtype == np.float64
            done = (term | trunc).cpu().numpy()
            ret = (ret.astype(np.float64) + r).astype(np.float32)   # float32 array += float64 rewards
            length = length + np.int32(1)
            assert np.array_equal(infos["_episode"].cpu().numpy(), done), t
            assert np.array_equal(infos["episode"]["r"].cpu().numpy()[done].view(np.int32), ret[done].view(np.int32)), t
            assert np.array_equal(infos["episode"]["l"].cpu().numpy()[done], length[done]), t
            count += int(done.sum())
            ret[done] = 0
            length[done] = 0
            assert np.array_equal(env.episode_returns.cpu().numpy().view(np.int32), ret.view(np.int32)), t
            assert np.array_equal(env.episode_lengths.cpu().numpy(), length), t
        assert env.episode_count == count > 0
        env.close()


def test_normalize_observation_and_reward():
    import gym_b200
    import torch
    from gym_b200.wrappers import NormalizeObservation, NormalizeReward
    N, T = 2048, 60
    base = gym_b200.vector.make("Pendulum-v1", N, max_episode_steps=25)
    twin = gym_b200.vector.make("Pendulum-v1", N, max_episode_steps=25)
    env = NormalizeReward(NormalizeObservation(base), gamma=0.9)
    o, _ = env.reset(seed=4)
    raw, _ = twin.reset(seed=4)
    mean, var, count = np.zeros(3), np.ones(3), 1e-4
    rmean, rvar, rcount = np.zeros(()), np.ones(()), 1e-4
    returns = np.zeros(N)
    x = raw.cpu().numpy().astype(np.float64)
    mean, var, count = _update_moments(mean, var, count, x)
    np.testing.assert_allclose(o.cpu().numpy(), (x - mean) / np.sqrt(var + 1e-8), rtol=2e-5, atol=2e-6)
    gen = torch.Generator(device="cuda").manual_seed(2)
    for t in range(T):
        a = torch.rand((N, 1), device="cuda", generator=gen) * 4 - 2
        o, r, te, tr, _ = env.step(a)
        raw, rr, rte, rtr, _ = twin.step(a)
        x = raw.cpu().numpy().astype(np.float64)
        mean, var, count = _update_moments(mean, var, count, x)                      # normalize.py:83-95
        np.testing.assert_allclose(o.cpu().numpy(), (x - mean) / np.sqrt(var + 1e-8), rtol=2e-5, atol=2e-6)
        rew = rr.cpu().numpy()
        returns = returns * 0.9 + rew                                                 # :130-144
        rmean, rvar, rcount = _update_moments(rmean, rvar, rcount, returns)
        np.testing.assert_allclose(r.cpu().numpy(), rew / np.sqrt(rvar + 1e-8), rtol=1e-9)
        returns[(rte | rtr).cpu().numpy()] = 0.0
        assert torch.equal(te, rte) and torch.equal(tr, rtr)
    np.testing.assert_allclose(env.env.obs_rms.mean.cpu().numpy(), mean, rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(env.env.obs_rms.var.cpu().numpy(), var, rtol=1e-9)
    np.testing.assert_allclose(env.return_rms.var.cpu().numpy()[0], rvar, rtol=1e-9)
    assert abs(float(env.env.obs_rms.count.item()) - count) < 1e-6
    env.close()
    twin.close()
