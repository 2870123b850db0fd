"""Per-env wrapper chains without a GPU: the numpy restatement against the reference fixture (and the live reference
where it is installed), the host build of csrc/subenv.cuh against the restatement, and the parsing of ``wrappers=``."""
import functools
import itertools
import os

import numpy as np
import pytest

from gym_b200 import subenv
from gym_b200.spaces import Box, Discrete
from conftest import GOLDEN
from hostsim import subenv_sim
from oracle import gen_subenv_fixtures as gen
from oracle.subenv_chain import SubenvChainRef

FIXTURE = os.path.join(GOLDEN, "reference", "subenv_wrappers.npz")
CASES = [(env_id, name) for env_id in gen.CLASSIC for name in ("ppo", "stats", "reordered")]


@pytest.fixture(scope="module")
def fixture():
    z = np.load(FIXTURE)
    return {k: z[k] for k in z.files}


def case(z, env_id, name):
    p = f"{env_id}/{name}/"
    return {k[len(p):]: v for k, v in z.items() if k.startswith(p)}


def stages_of(env_id, name):
    return gen.chains(env_id in ("MountainCarContinuous-v0", "Pendulum-v1"))[name]


def bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    assert a.dtype == b.dtype and a.shape == b.shape, (a.dtype, b.dtype, a.shape, b.shape)
    return np.array_equal(a.view(np.uint8), b.view(np.uint8))


def replay(c, env_id, name):
    """The restatement fed the raw run -> the wrapped run's arrays."""
    stages = stages_of(env_id, name)
    n, d = c["raw_obs0"].shape
    ref = SubenvChainRef([s.describe() for s in stages], env_id, n, d)
    out = {"obs0": ref.reset(c["raw_obs0"]), "obs": [], "reward": [], "final_obs": [], "episode_r": [],
           "episode_l": []}
    for t in range(c["raw_obs"].shape[0]):
        if t == gen.MID:
            out["obs_mid"] = ref.reset(c["raw_obs_mid"])
        o, r, fin, er, el = ref.step(c["raw_obs"][t], c["raw_reward"][t], c["raw_terminated"][t],
                                     c["raw_truncated"][t], c["raw_final_obs"][t])
        for k, v in zip(("obs", "reward", "final_obs", "episode_r", "episode_l"), (o, r, fin, er, el)):
            out[k].append(v)
    return {k: (np.stack(v) if isinstance(v, list) else v) for k, v in out.items()}


@pytest.mark.parametrize("env_id,name", CASES)
def test_restatement_equals_reference_fixture(fixture, env_id, name):
    c = case(fixture, env_id, name)
    assert np.array_equal(c["terminated"], c["raw_terminated"]) and np.array_equal(c["truncated"], c["raw_truncated"])
    done = c["terminated"] | c["truncated"]
    assert done.sum() >= 2 * c["obs"].shape[1], "the run must finish many episodes"
    out = replay(c, env_id, name)
    for k in ("obs0", "obs_mid", "obs", "reward"):
        assert bits_equal(out[k], c[k]), k
    normalized = any(isinstance(s, subenv.NormalizeObservation) for s in stages_of(env_id, name))
    assert np.array_equal(c["final_f64"], done & normalized)
    assert bits_equal(out["final_obs"][done].astype(np.float64), c["final_obs"][done])
    assert bits_equal(out["episode_r"], c["episode_r"]) and bits_equal(out["episode_l"], c["episode_l"])
    assert (c["episode_l"] >= 0).sum() == done.sum()


def test_episode_return_rounding_depends_on_reward_type(fixture):
    """MountainCarContinuous' Python-float rewards are rounded to float32 before the add: a float64 add would have
    given other returns in this fixture."""
    c = case(fixture, "MountainCarContinuous-v0", "stats")
    acc = np.zeros(c["raw_reward"].shape[1], np.float32)
    differ = 0
    for t in range(c["raw_reward"].shape[0]):
        if t == gen.MID:
            acc[:] = 0
        acc = (acc + c["raw_reward"][t]).astype(np.float32)
        done = c["terminated"][t] | c["truncated"][t]
        differ += int((acc[done] != c["episode_r"][t][done]).sum())
        acc[done] = 0
    assert differ > 0


@pytest.mark.parametrize("env_id,name", [("MountainCarContinuous-v0", "ppo"), ("CartPole-v1", "reordered"),
                                         ("Pendulum-v1", "stats")])
def test_fixture_equals_live_reference(fixture, env_id, name):
    from oracle.ref_gym import import_reference
    try:
        gym = import_reference()
    except ImportError:
        pytest.skip("the reference is not installed in oracle/_ref")
    wrapped, raw, acts = gen.run_case(gym, env_id, stages_of(env_id, name))
    c = case(fixture, env_id, name)
    assert bits_equal(acts, c["actions"])
    for k, v in wrapped.items():
        assert bits_equal(v, c[k]), k
    for k, v in raw.items():
        if f"raw_{k}" in c:
            assert bits_equal(v, c[f"raw_{k}"]), k


# ---- the host build of csrc/subenv.cuh against the restatement ---------------------------------------------------
STAGE_POOL = [subenv.RecordEpisodeStatistics(), subenv.NormalizeObservation(epsilon=1e-8),
              subenv.NormalizeReward(gamma=0.97, epsilon=1e-6), subenv.ClipObservation(-0.7, 1.3),
              subenv.ClipReward(-0.45, 0.9)]
# (id whose reward type the stream takes, kind, obs size)
STREAMS = [("CartPole-v1", 0, 4), ("Pendulum-v1", 3, 3), ("BipedalWalker-v3", 6, 24)]


def _orders():
    rng = np.random.default_rng(7)
    out = [list(p) for p in itertools.permutations(STAGE_POOL)][::17]
    for k in range(1, 5):
        for _ in range(3):
            out.append([STAGE_POOL[j] for j in rng.permutation(len(STAGE_POOL))[:k]])
    return out


ORDERS = _orders()


def _stream(rng, rtype, n, d, T):
    obs = (rng.standard_normal((T, n, d)) * rng.choice([0.1, 1.0, 30.0], size=(T, n, 1))).astype(np.float32)
    fin = (rng.standard_normal((T, n, d)) * 2).astype(np.float32)
    reward = rng.standard_normal((T, n)) * rng.choice([0.01, 1.0, 50.0], size=(T, n))
    reward[rng.random((T, n)) < 0.2] = 1.0
    if rtype == "f32":
        reward = reward.astype(np.float32).astype(np.float64)
    term = rng.random((T, n)) < 0.08
    trunc = rng.random((T, n)) < 0.04
    if rtype == "f32":   # BipedalWalker: most episodes end in a fall, whose reward is the Python int -100
        reward[term & (rng.random((T, n)) < 0.7)] = -100.0
    return obs, reward, term, trunc, fin


@pytest.mark.parametrize("env_id,kind,d", STREAMS)
@pytest.mark.parametrize("order", range(len(ORDERS)))
def test_host_build_equals_restatement(env_id, kind, d, order):
    stages = ORDERS[order]
    n, T = 64, 30
    chain = subenv.Chain(stages, kind, d, Discrete(2))
    host = subenv_sim.HostChain(chain, n)
    ref = SubenvChainRef([s.describe() for s in stages], env_id, n, d)
    rng = np.random.default_rng(order * 31 + kind)
    obs, reward, term, trunc, fin = _stream(rng, ref.raw_type, n, d, T)
    assert bits_equal(host.reset(obs[0]), ref.reset(obs[0]))
    for t in range(T):
        if t == T // 2:
            assert bits_equal(host.reset(obs[t]), ref.reset(obs[t]))
            continue
        ho, hr, hf32, hf64, her, hel = host.step(obs[t], reward[t], term[t], trunc[t], fin[t])
        ro, rr, rf, rer, rel = ref.step(obs[t], reward[t], term[t], trunc[t], fin[t])
        done = term[t] | trunc[t]
        assert bits_equal(ho, ro) and bits_equal(hr, rr), t
        hf = hf64 if chain.norm_obs else hf32
        assert bits_equal(hf[done], rf[done]), t
        assert bits_equal(her, rer) and bits_equal(hel, rel), t
    assert bits_equal(host.obs_stats[:d].T, ref.obs_mean) and bits_equal(host.rew_stats[3], ref.returns)


def test_clip_matches_numpy_on_edge_values():
    x = np.array([np.nan, -np.inf, np.inf, -0.0, 0.0, -1.0, 1.0, 0.5, -2.0, 2.0, 1e-45], np.float32)
    for lo, hi in ((-1.0, 1.0), (0.0, 1.0), (-0.0, 0.0), (-1.0, -1.0)):
        want = np.clip(x, np.float32(lo), np.float32(hi))
        assert bits_equal(subenv_sim.clip(x, lo, hi), want), (lo, hi)


# ---- parsing -----------------------------------------------------------------------------------------------------
def test_parse_accepts_specs_classes_and_single_wrappers():
    assert subenv.parse(None) is None and subenv.parse([]) is None
    assert subenv.parse(subenv.NormalizeObservation) == [subenv.NormalizeObservation()]
    assert subenv.parse(subenv.ClipReward(-1, 1)) == [subenv.ClipReward(-1.0, 1.0)]
    got = subenv.parse([subenv.RecordEpisodeStatistics, subenv.NormalizeReward(gamma=0.9)])
    assert got == [subenv.RecordEpisodeStatistics(100), subenv.NormalizeReward(0.9, 1e-8)]


def test_parse_accepts_the_reference_classes():
    from oracle.ref_gym import import_reference
    try:
        gym = import_reference()
    except ImportError:
        pytest.skip("the reference is not installed in oracle/_ref")
    w = gym.wrappers
    got = subenv.parse([w.RecordEpisodeStatistics, w.ClipAction, functools.partial(w.NormalizeObservation, epsilon=1e-6),
                        functools.partial(w.NormalizeReward, gamma=0.95)])
    assert got == [subenv.RecordEpisodeStatistics(), subenv.ClipAction(), subenv.NormalizeObservation(1e-6),
                   subenv.NormalizeReward(0.95)]
    for bad in (w.FrameStack, functools.partial(w.TransformObservation, f=lambda o: o),
                functools.partial(w.NormalizeReward, 0.9), functools.partial(w.NormalizeReward, beta=1.0)):
        with pytest.raises(ValueError):
            subenv.parse([bad])


@pytest.mark.parametrize("bad", [lambda e: e, "NormalizeObservation", subenv.ClipObservation, 3])
def test_parse_rejects_unsupported_wrappers(bad):
    with pytest.raises(ValueError, match="supported|bounds"):
        subenv.parse([bad])


def test_parse_rejects_repeats_and_bad_bounds():
    with pytest.raises(ValueError, match="twice"):
        subenv.parse([subenv.NormalizeObservation(), subenv.NormalizeObservation(epsilon=1e-3)])
    with pytest.raises(ValueError, match="low <= high"):
        subenv.ClipReward(1, -1)
    with pytest.raises(ValueError, match="low <= high"):
        subenv.ClipObservation(float("nan"), 1)


def test_chain_resolves_observation_bounds_and_raw_reward_types():
    box = Box(-1.0, 1.0, shape=(1,), dtype=np.float32)
    with pytest.raises(ValueError, match="Box"):
        subenv.Chain([subenv.ClipAction()], 0, 4, Discrete(2))
    c = subenv.Chain([subenv.RecordEpisodeStatistics(), subenv.ClipAction(), subenv.ClipObservation(-0.3, 0.3),
                      subenv.NormalizeObservation(), subenv.ClipReward(-0.7, 0.7)], 2, 2, box)
    assert c.clip_action and c.norm_obs and c.episode and not c.norm_reward and c.changes_rewards
    (ep, clip_obs, norm, clip_r) = c.ops
    assert clip_obs[1:] == (float(np.float32(-0.3)), float(np.float32(0.3)))   # float32 observation
    assert clip_r[1:] == (-0.7, 0.7)           # the kernel rounds them where the reward is an np.float32
    assert c.raw_reward_type == subenv.REWARD_PY and not c.int_reward_on_fall
    c = subenv.Chain([subenv.NormalizeObservation(), subenv.ClipObservation(-0.3, 0.3),
                      subenv.RecordEpisodeStatistics()], 6, 24, box)
    assert c.ops[1][1:] == (-0.3, 0.3) and not c.changes_rewards             # float64 observation
    assert c.raw_reward_type == subenv.REWARD_F32 and c.int_reward_on_fall
    assert subenv.Chain([subenv.RecordEpisodeStatistics()], 3, 3, box).raw_reward_type == subenv.REWARD_F64


def test_env_constructors_reject_bad_chains_before_touching_a_device():
    from gym_b200 import vector
    with pytest.raises(ValueError, match="Box"):
        vector.make("CartPole-v1", 4, wrappers=[subenv.ClipAction()])
    with pytest.raises(ValueError, match="autoreset"):
        vector.make("Pendulum-v1", 4, wrappers=[subenv.NormalizeObservation()], autoreset=False)
    with pytest.raises(ValueError, match="supported"):
        vector.make("Pendulum-v1", 4, wrappers=[lambda e: e])
    from gym_b200.env import B200Env
    with pytest.raises(ValueError, match="per-env wrappers"):
        B200Env("Pendulum-v1", wrappers=[subenv.NormalizeObservation()])


def _scripted_walker_streams(rng, n, T, d):
    """Per env: reset observations, and per step (obs, reward, terminated, truncated) with BipedalWalker's Python
    types: np.float32 rewards, the Python int -100 on a fall (bipedal_walker.py:598-600)."""
    steps = []
    for t in range(T):
        row = []
        for i in range(n):
            term, trunc = bool(rng.random() < 0.12), bool(rng.random() < 0.04)
            r = -100 if (term and rng.random() < 0.7) else np.float32(rng.standard_normal() * rng.choice([0.05, 3.0]))
            row.append(((rng.standard_normal(d) * 2).astype(np.float32), r, term, trunc))
        steps.append(row)
    resets = (rng.standard_normal((T + 1, n, d)) * 2).astype(np.float32)
    return steps, resets


def test_walker_fall_rewards_match_the_reference_wrappers():
    """The reference's own wrappers, in its SyncVectorEnv, over envs that replay BipedalWalker-typed outputs (np.float32
    rewards, the Python int -100 on a fall; the real walker needs Box2D): the restatement and the host build of
    csrc/subenv.cuh return the same, bit for bit, with reward-clip bounds that are not exact in float32."""
    from oracle.ref_gym import import_reference
    try:
        gym = import_reference()
    except ImportError:
        pytest.skip("the reference is not installed in oracle/_ref")
    n, T, d = 6, 80, 3
    steps, resets = _scripted_walker_streams(np.random.default_rng(11), n, T, d)

    class Replay(gym.Env):
        observation_space = gym.spaces.Box(-np.inf, np.inf, (d,), np.float32)
        action_space = gym.spaces.Discrete(2)

        def __init__(self, i):
            self.i, self.t, self.r = i, 0, 0

        def reset(self, seed=None, options=None):
            self.r += 1
            return resets[self.r - 1, self.i], {}

        def step(self, action):
            self.t += 1
            o, r, te, tr = steps[self.t - 1][self.i]
            return o, r, te, tr, {}

    chains = [[subenv.ClipReward(-0.7, 0.7), subenv.NormalizeReward(gamma=0.9), subenv.RecordEpisodeStatistics(),
               subenv.NormalizeObservation(), subenv.ClipObservation(-0.3, 0.3)],
              [subenv.RecordEpisodeStatistics(), subenv.ClipReward(-0.45, 0.9)],
              [subenv.NormalizeReward(), subenv.ClipReward(-0.45, 0.9), subenv.RecordEpisodeStatistics()]]
    falls = 0
    for stages in chains:
        wrappers = [gen.reference_wrapper(gym, s) for s in stages]

        def make(i):
            def thunk():
                e = Replay(i)
                for w in wrappers:
                    e = w(e)
                return e
            return thunk

        envs = gym.vector.SyncVectorEnv([make(i) for i in range(n)])
        ref = SubenvChainRef([s.describe() for s in stages], "BipedalWalker-v3", n, d)
        host = subenv_sim.HostChain(subenv.Chain(stages, 6, d, Discrete(2)), n)
        o, _ = envs.reset()
        assert bits_equal(ref.reset(resets[0]), o) and bits_equal(host.reset(resets[0]), o)
        k = np.ones(n, int)   # reset observations consumed per env
        for t in range(T):
            o, r, te, tr, info = envs.step(np.zeros(n, np.int64))
            done = te | tr
            raw_o = np.stack([resets[k[i], i] if done[i] else steps[t][i][0] for i in range(n)])
            raw_r = np.array([float(steps[t][i][1]) for i in range(n)])
            raw_f = np.stack([steps[t][i][0] for i in range(n)])
            k += done
            falls += int(sum(type(steps[t][i][1]) is int and done[i] for i in range(n)))
            ro, rr, rf, rer, rel = ref.step(raw_o, raw_r, te, tr, raw_f)
            ho, hr, hf32, hf64, her, hel = host.step(raw_o, raw_r, te, tr, raw_f)
            for got in ((ro, rr, rf, rer, rel), (ho, hr, hf64 if ref.normalizes_obs else hf32, her, hel)):
                assert bits_equal(got[0], o) and bits_equal(got[1], r), t
                for i in np.flatnonzero(done):
                    assert bits_equal(got[2][i].astype(info["final_observation"][i].dtype),
                                      info["final_observation"][i]), (t, i)
                    ep = info["final_info"][i]["episode"]
                    assert bits_equal(got[3][i], ep["r"]) and bits_equal(got[4][i], ep["l"]), (t, i)
        envs.close()
    assert falls > 20
