"""Reshaping per-env wrapper chains (FrameStack, TimeAwareObservation, FlattenObservation) and action stages
(ClipAction, RescaleAction) without a GPU: the numpy restatement against the reference fixture, the host build of
csrc/subenv.cuh against the restatement, the spaces the chain resolves, and the refusals."""
import functools
import os

import numpy as np
import pytest

from gym_b200 import subenv
from gym_b200.spaces import Box, Discrete
from conftest import GOLDEN
from hostsim import subenv_shapes_sim as sim
from oracle import gen_subenv_shape_fixtures as gen
from oracle.subenv_shapes import SubenvShapeRef, apply_actions

FIXTURE = os.path.join(GOLDEN, "reference", "subenv_shape_wrappers.npz")
CASES = [(env_id, name) for env_id, name, _ in gen.cases()]
KIND = {"CartPole-v1": 0, "MountainCar-v0": 1, "MountainCarContinuous-v0": 2, "Pendulum-v1": 3, "Acrobot-v1": 4}
RAW = {"CartPole-v1": (4, Discrete(2)), "MountainCar-v0": (2, Discrete(3)), "Acrobot-v1": (6, Discrete(3)),
       "MountainCarContinuous-v0": (2, Box(-1.0, 1.0, (1,), np.float32)),
       "Pendulum-v1": (3, Box(-2.0, 2.0, (1,), np.float32))}


@pytest.fixture(scope="module")
def fixture():
    z = np.load(FIXTURE)
    return {k: z[k] for k in z.files}


def case(z, env_id, name):
    return gen.load_case(z, env_id, name)


def stages_of(env_id, name):
    return {n: s for e, n, s in gen.cases() if e == env_id}[name]


def bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    assert a.dtype == b.dtype and a.shape == b.shape, (a.dtype, b.dtype, a.shape, b.shape)
    return np.array_equal(a.view(np.uint8), b.view(np.uint8))


def replay(c, env_id, name):
    """The restatement fed the raw run -> the wrapped run's arrays, in the output shape."""
    stages = stages_of(env_id, name)
    n, d = c["raw_obs0"].shape
    ref = SubenvShapeRef([s.describe() for s in stages], env_id, n, d)
    shape = (n,) + ref.shape
    out = {"obs0": ref.reset(c["raw_obs0"]).reshape(shape), "obs": [], "reward": [], "final_obs": [],
           "episode_r": [], "episode_l": []}
    for t in range(c["raw_obs"].shape[0]):
        if t == gen.MID:
            out["obs_mid"] = ref.reset(c["raw_obs_mid"]).reshape(shape)
        o, r, fin, er, el = ref.step(c["raw_obs"][t], c["raw_reward"][t], c["raw_terminated"][t],
                                     c["raw_truncated"][t], c["raw_final_obs"][t])
        for k, v in zip(("obs", "reward", "final_obs", "episode_r", "episode_l"),
                        (o.reshape(shape), r, fin.reshape(shape), er, el)):
            out[k].append(v)
    return ref, {k: (np.stack(v) if isinstance(v, list) else v) for k, v in out.items()}


@pytest.mark.parametrize("env_id,name", CASES)
def test_restatement_equals_reference_fixture(fixture, env_id, name):
    c = case(fixture, env_id, name)
    assert np.array_equal(c["terminated"], c["raw_terminated"]) and np.array_equal(c["truncated"], c["raw_truncated"])
    done = c["terminated"] | c["truncated"]
    assert done.sum() >= 2 * c["obs"].shape[1], "the run must finish many episodes"
    ref, out = replay(c, env_id, name)
    for k in ("obs0", "obs_mid", "obs", "reward"):
        assert bits_equal(out[k], c[k]), k
    assert np.array_equal(c["final_f64"], done & (ref.final_dtype == np.float64))
    assert bits_equal(out["final_obs"][done].astype(np.float64), c["final_obs"][done])
    assert bits_equal(out["episode_r"], c["episode_r"]) and bits_equal(out["episode_l"], c["episode_l"])


def test_time_aware_terminal_rows_end_in_the_episode_length(fixture):
    c = case(fixture, "CartPole-v1", "time")
    done = c["terminated"] | c["truncated"]
    last = c["final_obs"][done][:, -1]
    assert c["final_f64"][done].all() and (last >= 1).all() and (last <= gen.MAX_STEPS).all()
    assert (last == gen.MAX_STEPS).any() and (c["obs0"][:, -1] == 0).all()


@pytest.mark.parametrize("env_id,name", [(e, n) for e, n in CASES if e in gen.CONTINUOUS])
def test_action_stages_equal_the_reference(fixture, env_id, name):
    """The restatement and the host build of the action kernel give the actions the reference's wrappers gave."""
    c = case(fixture, env_id, name)
    stages = stages_of(env_id, name)
    d, space = RAW[env_id]
    want = c["raw_actions"]
    got = apply_actions([s.describe() for s in stages], space.low, space.high, c["actions"])
    assert bits_equal(got, want)
    chain = subenv.Chain(stages, KIND[env_id], d, space)
    assert bits_equal(sim.actions(chain, c["actions"].reshape(-1, 1)).reshape(want.shape), want)
    if any(isinstance(s, subenv.ClipAction) for s in stages) or name == "rescale":
        assert not bits_equal(c["actions"], want)


@pytest.mark.parametrize("env_id,name", CASES)
def test_chain_spaces_equal_the_reference(fixture, env_id, name):
    c = case(fixture, env_id, name)
    d, space = RAW[env_id]
    from gym_b200 import envs as _envs
    kind = KIND[env_id]
    params = _envs.resolve_params(kind, {})
    obs_space, act_space = _envs.KINDS[kind].spaces(params)
    chain = subenv.Chain(stages_of(env_id, name), kind, d, act_space, obs_space)
    o = chain.observation_space
    assert o.dtype == np.float32   # the reference's are float32 (the fixture's generator checks)
    assert bits_equal(o.low, c["obs_low"]) and bits_equal(o.high, c["obs_high"])
    assert chain.obs_shape == c["obs"].shape[2:] == o.shape
    if "act_low" in c:
        a = chain.action_space
        assert a.dtype == np.float32 and bits_equal(a.low, c["act_low"]) and bits_equal(a.high, c["act_high"])


# ---- the host build of csrc/subenv.cuh against the restatement ---------------------------------------------------
SHAPE_CHAINS = {
    "fs4": [subenv.FrameStack(4)],
    "norm_fs3_clip": [subenv.NormalizeObservation(), subenv.FrameStack(3), subenv.ClipObservation(-0.6, 0.8)],
    "fs2_norm": [subenv.FrameStack(2), subenv.NormalizeObservation(epsilon=1e-6)],
    "time": [subenv.TimeAwareObservation()],
    "time_norm": [subenv.TimeAwareObservation(), subenv.NormalizeObservation(), subenv.ClipObservation(-2, 2)],
    "time_fs3": [subenv.RecordEpisodeStatistics(), subenv.TimeAwareObservation(), subenv.FrameStack(3)],
    "fs2_time_flat": [subenv.FrameStack(2), subenv.TimeAwareObservation(), subenv.FlattenObservation()],
    "norm_flat": [subenv.NormalizeObservation(), subenv.FlattenObservation(), subenv.ClipObservation(-0.3, 0.3)],
    "ppo_all": [subenv.RecordEpisodeStatistics(), subenv.NormalizeObservation(), subenv.ClipObservation(-10, 10),
                subenv.NormalizeReward(gamma=0.97), subenv.ClipReward(-0.45, 0.9), subenv.TimeAwareObservation(),
                subenv.FrameStack(4), subenv.FlattenObservation()],
    "fs1": [subenv.FrameStack(1), subenv.NormalizeObservation()],
}
STREAMS = [("CartPole-v1", 0, 4), ("Pendulum-v1", 3, 3), ("BipedalWalker-v3", 6, 24)]


def _stream(rng, rtype, n, d, T):
    obs = (rng.standard_normal((T, n, d)) * rng.choice([0.1, 1.0, 30.0], size=(T, n, 1))).astype(np.float32)
    fin = (rng.standard_normal((T, n, d)) * 2).astype(np.float32)
    reward = rng.standard_normal((T, n)) * rng.choice([0.01, 1.0, 50.0], size=(T, n))
    if rtype == "f32":
        reward = reward.astype(np.float32).astype(np.float64)
    term = rng.random((T, n)) < 0.08
    trunc = rng.random((T, n)) < 0.04
    if rtype == "f32":   # BipedalWalker: most episodes end in a fall, whose reward is the Python int -100
        reward[term & (rng.random((T, n)) < 0.7)] = -100.0
    return obs, reward, term, trunc, fin


@pytest.mark.parametrize("env_id,kind,d", STREAMS)
@pytest.mark.parametrize("name", list(SHAPE_CHAINS))
def test_host_build_equals_restatement(env_id, kind, d, name):
    stages = SHAPE_CHAINS[name]
    n, T = 48, 40
    chain = subenv.Chain(stages, kind, d, Discrete(2))
    host = sim.HostShapeChain(chain, n)
    ref = SubenvShapeRef([s.describe() for s in stages], env_id, n, d)
    assert ref.shape == chain.obs_shape and ref.width == host.W
    shape = (n,) + ref.shape
    rng = np.random.default_rng(len(name) * 131 + kind)
    obs, reward, term, trunc, fin = _stream(rng, ref.raw_type, n, d, T)
    assert bits_equal(host.reset(obs[0]), ref.reset(obs[0]).reshape(shape))
    for t in range(T):
        if t == T // 2:
            assert bits_equal(host.reset(obs[t]), ref.reset(obs[t]).reshape(shape))
            continue
        ho, hr, hf, her, hel = host.step(obs[t], reward[t], term[t], trunc[t], fin[t])
        ro, rr, rf, rer, rel = ref.step(obs[t], reward[t], term[t], trunc[t], fin[t])
        done = term[t] | trunc[t]
        assert bits_equal(ho, ro.reshape(shape)) and bits_equal(hr, rr), t
        assert bits_equal(hf[done], rf.reshape(shape)[done]), t
        assert bits_equal(her, rer) and bits_equal(hel, rel), t
    if ref.t is not None:
        assert bits_equal(host.t, ref.t)


def test_host_build_normalize_variance_follows_the_dtype():
    """A float64 value beyond float32's range after TimeAwareObservation: (x - x)**2 in float64 is 0, in float32 NaN."""
    stages = [subenv.TimeAwareObservation(), subenv.NormalizeObservation()]
    chain = subenv.Chain(stages, 3, 3, Discrete(2))
    host = sim.HostShapeChain(chain, 2)
    ref = SubenvShapeRef([s.describe() for s in stages], "Pendulum-v1", 2, 3)
    big = np.full((2, 3), 3e38, np.float32)
    assert bits_equal(host.reset(big), ref.reset(big).reshape(2, 4))
    zero = np.zeros(2)
    for _ in range(3):
        ho, *_ = host.step(big, zero, [0, 0], [0, 0], big)
        ro, *_ = ref.step(big, zero, [0, 0], [0, 0], big)
        assert bits_equal(ho, ro.reshape(2, 4))
    assert np.isfinite(host.obs_stats[4:8]).all()


def test_host_action_stages_on_edge_values():
    x = np.array([[np.nan], [-np.inf], [np.inf], [-0.0], [0.0], [-1.0], [1.0], [0.5], [-2.0], [2.0], [1e-45]],
                 np.float32)
    box = Box(-2.0, 2.0, (1,), np.float32)
    for stages in ([subenv.RescaleAction(-1, 1)], [subenv.ClipAction(), subenv.RescaleAction(-1, 1)],
                   [subenv.RescaleAction(-1, 1), subenv.ClipAction()],
                   [subenv.RescaleAction(np.float32(-0.3), np.array([0.7], np.float32))]):
        chain = subenv.Chain(stages, 3, 3, box)
        with np.errstate(invalid="ignore"):
            want = apply_actions([s.describe() for s in stages], box.low, box.high, x)
        assert bits_equal(sim.actions(chain, x), want), stages


# ---- parsing, spaces and refusals --------------------------------------------------------------------------------
def test_parse_accepts_the_new_stages():
    got = subenv.parse([subenv.TimeAwareObservation, subenv.FlattenObservation, subenv.FrameStack(4),
                        subenv.RescaleAction(-1, 1)])
    assert got == [subenv.TimeAwareObservation(), subenv.FlattenObservation(), subenv.FrameStack(4),
                   subenv.RescaleAction(-1.0, 1.0)]
    assert subenv.FrameStack(4).describe() == ["FrameStack", {"num_stack": 4.0}]
    assert subenv.RescaleAction(-1, np.array([0.5, 2], np.float32)).describe() == \
        ["RescaleAction", {"max_action": [0.5, 2.0], "min_action": -1.0}]
    # the descriptions of the stages that existed before are unchanged
    assert subenv.NormalizeObservation().describe() == ["NormalizeObservation", {"epsilon": 1e-8}]
    assert subenv.ClipAction().describe() == ["ClipAction", {}]


def test_parse_accepts_the_reference_classes():
    from oracle.ref_gym import import_reference
    try:
        gym = import_reference()
    except ImportError:
        pytest.skip("the reference is not installed in oracle/_ref")
    w = gym.wrappers
    got = subenv.parse([w.TimeAwareObservation, functools.partial(w.FrameStack, num_stack=3), w.FlattenObservation,
                        functools.partial(w.RescaleAction, min_action=-1, max_action=1.0)])
    assert got == [subenv.TimeAwareObservation(), subenv.FrameStack(3), subenv.FlattenObservation(),
                   subenv.RescaleAction(-1, 1)]
    for bad in (w.FrameStack, w.RescaleAction, functools.partial(w.FrameStack, 3),
                functools.partial(w.RescaleAction, -1, 1),
                functools.partial(w.FrameStack, num_stack=3, lz4_compress=True)):
        with pytest.raises(ValueError):
            subenv.parse([bad])


@pytest.mark.parametrize("num_stack", [0, -1, subenv.MAX_STACK + 1, 2.0, True])
def test_frame_stack_refuses_bad_num_stack(num_stack):
    with pytest.raises(ValueError, match="num_stack"):
        subenv.FrameStack(num_stack)


def test_frame_stack_refuses_lz4():
    with pytest.raises(ValueError, match="lz4"):
        subenv.FrameStack(4, lz4_compress=True)


def test_rescale_action_refuses_discrete_kinds():
    with pytest.raises(ValueError, match="Box"):
        subenv.Chain([subenv.RescaleAction(-1, 1)], 0, 4, Discrete(2))


@pytest.mark.parametrize("bound", [np.float64(1.0), np.array([1.0]), np.int64(1), [1.0], np.array([1], np.int32),
                                   np.array([[1.0]], np.float32)])
def test_rescale_action_refuses_bounds_that_make_the_actions_float64(bound):
    with pytest.raises(ValueError, match="float64|float32"):
        subenv.RescaleAction(-1, bound)


def test_rescale_action_refuses_min_above_max():
    with pytest.raises(ValueError, match="min_action <= max_action"):
        subenv.RescaleAction(1, -1)
    with pytest.raises(ValueError, match="min_action <= max_action"):
        subenv.RescaleAction(np.array([-1, 2], np.float32), np.array([1, 1], np.float32))
    with pytest.raises(ValueError, match="min_action <= max_action"):
        subenv.RescaleAction(float("nan"), 1)


def test_rescale_action_refuses_a_bound_of_another_shape():
    with pytest.raises(ValueError, match="action shape"):
        subenv.Chain([subenv.RescaleAction(np.zeros(2, np.float32), 1)], 3, 3, Box(-2.0, 2.0, (1,), np.float32))


def test_repeated_new_stages_are_refused():
    for s in (subenv.FrameStack(2), subenv.TimeAwareObservation(), subenv.FlattenObservation(),
              subenv.RescaleAction(-1, 1)):
        with pytest.raises(ValueError, match="twice"):
            subenv.parse([s, s])


def test_chain_resolves_widths_dtypes_and_state():
    c = subenv.Chain([subenv.NormalizeObservation(), subenv.TimeAwareObservation(), subenv.FrameStack(3)], 6, 24,
                     Box(-1.0, 1.0, (4,), np.float32))
    assert c.obs_shape == (3, 25) and c.out_width == 75 and c.final_f64 and c.reshape
    assert c.stack == (3, 25, True) and c.time_aware and c.norm_width == 24
    c = subenv.Chain([subenv.FrameStack(2), subenv.NormalizeObservation(), subenv.FlattenObservation()], 0, 4,
                     Discrete(2))
    assert c.obs_shape == (8,) and not c.final_f64 and c.norm_width == 8 and c.stack == (2, 4, False)
    c = subenv.Chain([subenv.NormalizeObservation(), subenv.ClipObservation(-5, 5)], 0, 4, Discrete(2))
    assert not c.reshape and c.obs_shape == (4,) and c.final_f64 == c.norm_obs


def test_sample_plan_follows_the_rescaled_space():
    """sample_actions draws from the chain's action space, so a rescaled Box samples in [min, max]."""
    c = subenv.Chain([subenv.ClipAction(), subenv.RescaleAction(np.float32(-0.25), 0.5)], 3, 3,
                     Box(-2.0, 2.0, (1,), np.float32))
    from gym_b200.spaces import batch_space
    space = batch_space(c.action_space, n=4096)
    space.seed(5)
    x = space.sample()
    assert x.dtype == np.float32 and x.min() >= np.float32(-0.25) and x.max() <= np.float32(0.5)
    assert bits_equal(c.action_space.low, np.array([-0.25], np.float32))
