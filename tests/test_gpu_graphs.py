"""CUDA graph capture of ``B200VectorEnv.step()``, ``reset()`` and ``sample_actions()`` (DESIGN §4.8): replay k gives,
bit for bit, what the k-th eager call gives on an identically seeded twin fed the same actions, and every operation
that cannot be captured raises ``error.Error`` without harming the env."""
import copy

import numpy as np
import pytest

from oracle import ref_gym

pytestmark = pytest.mark.gpu
needs_reference = pytest.mark.skipif(ref_gym.reference_path() is None,
                                     reason="the reference is not installed in oracle/_ref")

IDS = ["CartPole-v0", "CartPole-v1", "MountainCar-v0", "MountainCarContinuous-v0", "Pendulum-v1", "Acrobot-v1",
       "LunarLander-v2", "LunarLanderContinuous-v2", "BipedalWalker-v3", "BipedalWalkerHardcore-v3"]
BOX2D = ("LunarLander", "BipedalWalker")


def _torch():
    import torch
    return torch


def _make(env_id, n, **kw):
    import gym_b200
    return gym_b200.vector.make(env_id, n, device=0, **kw)


def _pair(env_id, n, seed=5, **kw):
    a, b = _make(env_id, n, **kw), _make(env_id, n, **kw)
    a.reset(seed=seed)
    b.reset(seed=seed)
    return a, b


class _Actions:
    """A seeded stream of action batches for `env` (torch generator on the device): out-of-bounds Box actions
    included, so the kernels' own clipping is exercised."""

    def __init__(self, env, seed=0):
        torch = _torch()
        self.env = env
        self.g = torch.Generator(device="cuda:0")
        self.g.manual_seed(seed)

    def next(self, dtype=None):
        torch, e = _torch(), self.env
        if e.discrete:
            a = torch.randint(0, int(e.single_action_space.n), (e.num_envs,), generator=self.g, device="cuda:0")
            return a if dtype is None else a.to(dtype)
        lo = torch.as_tensor(e.single_action_space.low, device="cuda:0")
        hi = torch.as_tensor(e.single_action_space.high, device="cuda:0")
        u = torch.rand((e.num_envs, e.act_dim), generator=self.g, device="cuda:0", dtype=torch.float32)
        return lo - 0.2 * (hi - lo) + 1.4 * (hi - lo) * u


def _capture(fn):
    torch = _torch()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = fn()
    return g, out


def _flat(step_out):
    """The tensors of one step's results that the contract covers."""
    obs, rew, term, trunc, infos = step_out
    out = {"obs": obs, "reward": rew, "terminated": term, "truncated": trunc,
           "final_observation": infos["final_observation"], "_final_observation": infos["_final_observation"]}
    if "final_info" in infos:
        out["_final_info"] = infos["_final_info"]
        out["episode_r"] = infos["final_info"]["episode"]["r"]
        out["episode_l"] = infos["final_info"]["episode"]["l"]
    if "episode" in infos:   # gym_b200.wrappers.RecordEpisodeStatistics
        out["w_episode_r"] = infos["episode"]["r"]
        out["w_episode_l"] = infos["episode"]["l"]
        out["w_episode_mask"] = infos["_episode"]
    return out


def _bits(t):
    torch = _torch()
    if t.dtype in (torch.float32, torch.int32):
        return t.view(torch.int32)
    if t.dtype in (torch.float64, torch.int64):
        return t.view(torch.int64)
    return t


# results whose rows are valid only where a mask is set; the others hold whatever the buffer held (a graph always
# writes the same buffers, eager steps alternate between two sets)
_MASKED = {"final_observation": "_final_observation", "episode_r": "_final_info", "episode_l": "_final_info",
           "w_episode_r": "w_episode_mask", "w_episode_l": "w_episode_mask"}


def _assert_same(got, want, what):
    """Bitwise equality (masked results in their valid rows)."""
    assert got.keys() == want.keys(), what
    for k in want:
        g, w = got[k], want[k]
        assert g.dtype == w.dtype and g.shape == w.shape, (what, k, g.dtype, w.dtype, g.shape, w.shape)
        if k in _MASKED:
            mask = want[_MASKED[k]]
            assert _torch().equal(got[_MASKED[k]], mask), (what, k)
            g, w = g[mask], w[mask]
        if not _torch().equal(_bits(g), _bits(w)):
            bad = (_bits(g) != _bits(w)).nonzero()
            raise AssertionError(f"{what}: {k} differs in {len(bad)} entries, first at {bad[0].tolist()}")


def _assert_same_rows(a, b):
    _torch().cuda.synchronize()
    assert _torch().equal(a.snapshot().rows, b.snapshot().rows)


# ---------------------------------------------------------------------------------------------- one captured step
@pytest.mark.parametrize("env_id", IDS)
def test_captured_step_matches_eager(env_id):
    """One captured step, its action buffer refilled between replays: every replay equals the twin's eager step, and
    the two envs' whole state agrees at the end."""
    box2d = env_id.startswith(BOX2D)
    n, replays = (1 << 12, 100) if box2d else (2048, 300)
    a, b = _pair(env_id, n)
    gen = _Actions(a, seed=1)
    act = gen.next().clone()
    graph, out = _capture(lambda: _flat(a.step(act)))
    for k in range(replays):
        act.copy_(gen.next())
        graph.replay()
        _assert_same(out, _flat(b.step(act)), f"{env_id} replay {k}")
    _assert_same_rows(a, b)
    a.close(), b.close()


# ---------------------------------------------------------------------------- the first step of a handle captured
def _first_step_cases():
    cases = [("CartPole-v1", 1 << 20, dt) for dt in ("int64", "int32", "uint8")]   # kernel B
    cases += [(i, 1 << 16, dt) for i in ("MountainCar-v0", "Acrobot-v1") for dt in ("int64", "int32", "uint8")]
    cases += [(i, 1 << 16, "float32") for i in ("MountainCarContinuous-v0", "Pendulum-v1")]   # kernel P
    cases += [("LunarLander-v2", 1 << 12, dt) for dt in ("int64", "int32", "uint8")]
    cases += [(i, 1 << 12, "float32") for i in ("LunarLanderContinuous-v2", "BipedalWalker-v3")]
    return cases


@pytest.mark.parametrize("env_id,n,dtype", _first_step_cases())
def test_first_step_of_a_handle_captured(env_id, n, dtype):
    """No eager step (of this handle, or of this action dtype) before the capture: the kernels' launch set-up happens
    when the handle is created, so the captured first step is a plain launch."""
    torch = _torch()
    a, b = _pair(env_id, n, seed=12)
    gen = _Actions(a, seed=2)
    act = gen.next(getattr(torch, dtype)).clone()
    graph, out = _capture(lambda: _flat(a.step(act)))
    for k in range(10):
        act.copy_(gen.next(getattr(torch, dtype)))
        graph.replay()
        _assert_same(out, _flat(b.step(act)), f"{env_id} {dtype} replay {k}")
    _assert_same_rows(a, b)
    a.close(), b.close()


# ---------------------------------------------------------------------------------------- per-env wrapper chains
def _full_chain():
    from gym_b200 import subenv
    return [subenv.RecordEpisodeStatistics(), subenv.RescaleAction(-1.0, 1.0), subenv.ClipAction(),
            subenv.NormalizeObservation(), subenv.NormalizeReward(), subenv.FrameStack(4),
            subenv.TimeAwareObservation(), subenv.FlattenObservation()]


def _discrete_chain():
    from gym_b200 import subenv
    return [subenv.RecordEpisodeStatistics(), subenv.FrameStack(2), subenv.NormalizeObservation(),
            subenv.NormalizeReward()]


@pytest.mark.parametrize("env_id,chain", [("Pendulum-v1", _full_chain), ("LunarLanderContinuous-v2", _full_chain),
                                          ("CartPole-v1", _discrete_chain)])
def test_captured_step_through_a_wrapper_chain(env_id, chain):
    """Final observations (float32, and the float64 rows of the Discrete chain), the done masks read after the
    replays, and final_info's episode r / l; infos["final_info"]["episode"]["t"] keeps its capture-time value."""
    a, b = (_make(env_id, 1024, wrappers=chain(), max_episode_steps=40) for _ in range(2))
    a.reset(seed=3)
    b.reset(seed=3)
    if chain is _discrete_chain:
        assert a._chain.final_f64
    gen = _Actions(a, seed=4)
    act = gen.next().clone()
    infos = {}

    def step():
        r = a.step(act)
        infos["t"] = r[4]["final_info"]["episode"]["t"]
        infos["d"] = r[4]
        return _flat(r)
    graph, out = _capture(step)
    dones = 0
    for k in range(120):
        act.copy_(gen.next())
        graph.replay()
        want = _flat(b.step(act))
        _assert_same(out, want, f"{env_id} replay {k}")
        dones += int(want["_final_observation"].sum())
        assert infos["d"]["final_info"]["episode"]["t"] == infos["t"]
    assert dones > 0
    _assert_same_rows(a, b)
    a.close(), b.close()


# --------------------------------------------------------------------------------- a graph of steps and a policy
def test_graph_of_eight_steps_with_a_policy():
    """8 steps with a policy computed from each observation, behind the vector RecordEpisodeStatistics wrapper,
    replayed 20 times, against 160 eager steps of the twin."""
    torch = _torch()
    from gym_b200 import wrappers
    n = 4096
    a = wrappers.RecordEpisodeStatistics(_make("CartPole-v1", n))
    b = wrappers.RecordEpisodeStatistics(_make("CartPole-v1", n))
    obs_a, _ = a.reset(seed=8)
    obs_b, _ = b.reset(seed=8)
    # pushes the pole the way it leans: episodes end within a few dozen steps
    w = torch.tensor([0.1, 0.5, -2.0, -0.7], dtype=torch.float32, device="cuda:0")
    state = obs_a.clone()   # the graph's input: the last observation

    def policy(obs):
        return ((obs * w).sum(-1) > 0).to(torch.int64)

    def rollout():
        steps, obs = [], state
        for _ in range(8):
            r = a.step(policy(obs))
            steps.append({k: v.clone() for k, v in _flat(r).items()})
            obs = r[0]
        state.copy_(obs)
        return steps
    graph, steps = _capture(rollout)
    obs = obs_b
    for rep in range(20):
        graph.replay()
        for k in range(8):
            r = b.step(policy(obs))
            _assert_same(steps[k], _flat(r), f"replay {rep} step {k}")
            obs = r[0]
    # (the ring behind return_queue takes episodes that end in the same step in the order their threads reach its
    # counter, so only the count is compared; each step's episode r / l were compared above)
    assert a.episode_count == b.episode_count and a.episode_count > 0
    _assert_same_rows(a.unwrapped, b.unwrapped)
    a.close(), b.close()


# -------------------------------------------------------------------------------------------- sample_actions()
def _pcg(space):
    return space.np_random.bit_generator.state


@pytest.mark.parametrize("env_id", ["CartPole-v1", "BipedalWalker-v3"])
def test_captured_sample_and_step(env_id):
    """Replays of step(sample_actions()) draw the twin's eager sample_actions() sequence; sync_action_space() then
    brings the host generator to the twin's."""
    n = 1 << 12
    a, b = _pair(env_id, n, seed=2)
    a.action_space.seed(9)
    b.action_space.seed(9)
    _assert_same({"a": a.sample_actions()}, {"a": b.sample_actions()}, "eager draw")   # puts the stream on the device
    holder = {}

    def step():
        holder["act"] = a.sample_actions()
        return _flat(a.step(holder["act"]))
    host_before = _pcg(a.action_space)
    graph, out = _capture(step)
    assert _pcg(a.action_space) == host_before      # the capture leaves the host generator alone
    for k in range(25):
        graph.replay()
        bact = b.sample_actions()
        _assert_same({"a": holder["act"]}, {"a": bact}, f"actions, replay {k}")
        _assert_same(out, _flat(b.step(bact)), f"step, replay {k}")
    assert _pcg(a.action_space) == host_before
    a.sync_action_space()
    assert _pcg(a.action_space) == _pcg(b.action_space)
    # and eager and captured draws keep interleaving
    _assert_same({"a": a.sample_actions()}, {"a": b.sample_actions()}, "eager after sync")
    graph.replay()
    bact = b.sample_actions()
    _assert_same({"a": holder["act"]}, {"a": bact}, "replay after sync")
    _assert_same(out, _flat(b.step(bact)), "step, replay after sync")
    _assert_same_rows(a, b)
    a.close(), b.close()


def test_host_draws_and_reseeds_after_a_capture():
    """DESIGN §4.8: replays advance the device stream only; an eager sample_actions() continues it while the host
    generator is where sample_actions() left it, and follows the host generator once it was drawn from or reseeded."""
    n = 3000
    env = _make("Pendulum-v1", n)
    env.reset(seed=0)
    env.action_space.seed(21)
    ref = copy.deepcopy(env.action_space)   # the stream the device follows
    np.testing.assert_array_equal(env.sample_actions().cpu().numpy(), ref.sample())
    holder = {}
    graph, _ = _capture(lambda: holder.setdefault("x", env.sample_actions()))
    for _ in range(3):
        graph.replay()
        np.testing.assert_array_equal(holder["x"].cpu().numpy(), ref.sample())
    # eager, host untouched: the device stream goes on (the host generator is 3 batches behind it)
    np.testing.assert_array_equal(env.sample_actions().cpu().numpy(), ref.sample())
    # a host draw: the next eager call starts from the host generator, and the replays follow it
    env.action_space.sample()
    host = copy.deepcopy(env.action_space)
    np.testing.assert_array_equal(env.sample_actions().cpu().numpy(), host.sample())
    graph.replay()
    np.testing.assert_array_equal(holder["x"].cpu().numpy(), host.sample())
    # a reseed (another inc): the same
    env.action_space.seed(2 ** 80 + 1)
    host = copy.deepcopy(env.action_space)
    np.testing.assert_array_equal(env.sample_actions().cpu().numpy(), host.sample())
    graph.replay()
    graph.replay()
    host.sample()
    np.testing.assert_array_equal(holder["x"].cpu().numpy(), host.sample())
    env.sync_action_space()
    assert _pcg(env.action_space) == _pcg(host)
    env.close()


def test_two_draws_in_one_graph_are_consecutive():
    env = _make("CartPole-v1", 5000)
    env.reset(seed=0)
    env.action_space.seed(4)
    ref = copy.deepcopy(env.action_space)
    np.testing.assert_array_equal(env.sample_actions().cpu().numpy(), ref.sample())
    graph, (x, y) = _capture(lambda: (env.sample_actions(), env.sample_actions()))
    for _ in range(4):
        graph.replay()
        np.testing.assert_array_equal(x.cpu().numpy(), ref.sample())
        np.testing.assert_array_equal(y.cpu().numpy(), ref.sample())
    env.close()


def test_sample_capture_before_an_eager_draw_is_refused():
    from gym_b200 import error
    torch = _torch()
    env = _make("CartPole-v1", 64)
    env.reset(seed=0)
    torch.cuda.synchronize()
    with pytest.raises(error.Error, match="outside the capture"):
        with torch.cuda.graph(torch.cuda.CUDAGraph()):
            env.sample_actions()
    env.action_space.seed(1)
    ref = copy.deepcopy(env.action_space)
    np.testing.assert_array_equal(env.sample_actions().cpu().numpy(), ref.sample())
    env.close()


# ----------------------------------------------------------------------------------------------- captured reset
@pytest.mark.parametrize("env_id,options", [("CartPole-v1", None), ("MountainCar-v0", {"low": -0.6, "high": -0.5}),
                                            ("LunarLander-v2", None)])
def test_captured_reset_then_steps(env_id, options):
    """reset(seed=s) and 6 steps in one graph: every replay gives the same trajectory as the twin's eager run."""
    torch = _torch()
    n = 1024
    a, b = _make(env_id, n), _make(env_id, n)
    a.reset(seed=1)
    gen = _Actions(a, seed=6)
    acts = [gen.next() for _ in range(6)]

    def run(env):
        steps = [{"obs": env.reset(seed=33, options=options)[0].clone()}]
        for act in acts:
            steps.append({k: v.clone() for k, v in _flat(env.step(act)).items()})
        return steps
    graph, got = _capture(lambda: run(a))
    for rep in range(3):
        graph.replay()
        want = run(b)
        for k in range(len(want)):
            _assert_same(got[k], want[k], f"replay {rep} entry {k}")
    torch.cuda.synchronize()
    _assert_same_rows(a, b)
    a.close(), b.close()


# ------------------------------------------------------------------------------------------------------ refusals
def _refused(fn, match):
    from gym_b200 import error
    torch = _torch()
    torch.cuda.synchronize()
    with pytest.raises(error.Error, match=match):
        with torch.cuda.graph(torch.cuda.CUDAGraph()):
            fn()


def _steps_like_twin(a, b, steps=5, seed=0):
    gen = _Actions(a, seed=seed)
    for k in range(steps):
        act = gen.next()
        _assert_same(_flat(a.step(act)), _flat(b.step(act)), f"eager step {k} after a refusal")


def test_refusals_leave_the_env_stepping_like_its_twin():
    from gym_b200 import wrappers
    torch = _torch()
    a, b = _pair("CartPole-v1", 256, seed=4)
    act = torch.zeros(256, dtype=torch.int64, device="cuda:0")
    _refused(lambda: a.step(np.zeros(256, dtype=np.int64)), "not a CUDA tensor")
    host_act = act.cpu()
    _refused(lambda: a.step(host_act), "not a CUDA tensor")
    _refused(lambda: a.reset(seed=list(range(256))), r"reset\(seed=<list>\)")
    _refused(lambda: a.seed(list(range(256))), r"seed\(<list>\)")
    _refused(lambda: a.snapshot(), r"snapshot\(\)")
    snap = b.snapshot()
    _refused(lambda: a.restore(snap), r"restore\(\)")
    _refused(lambda: a.clone(torch.arange(256, device="cuda:0")), r"clone\(\)")
    _refused(lambda: a.check_actions(), r"check_actions\(\)")
    _refused(lambda: a.set_state(elapsed=np.zeros(256, np.int32)), r"set_state\(\)")
    _refused(lambda: a.sync_action_space(), r"sync_action_space\(\)")
    _steps_like_twin(a, b)
    # wrappers whose state is steered from the host
    for cls in (wrappers.NormalizeObservation, wrappers.NormalizeReward, wrappers.VectorListInfo):
        w = cls(a)
        _refused(lambda: w.step(act), cls.__name__)
        _refused(lambda: w.reset(seed=2), cls.__name__)
    _steps_like_twin(a, b, seed=1)
    _assert_same_rows(a, b)
    a.close(), b.close()


def test_refusals_of_host_backends():
    import gym_b200
    from gym_b200.distributed import ShardedVectorEnv
    a, b = _pair("Acrobot-v1", 128, seed=6, backend="numpy")
    _refused(lambda: a.step(np.zeros(128, dtype=np.int64)), "backend='numpy'")
    _refused(lambda: a.reset(seed=1), "backend='numpy'")
    _refused(lambda: a.sample_actions(), "backend='numpy'")
    for k in range(4):
        x = np.full(128, k % 3, dtype=np.int64)
        ra, rb = a.step(x), b.step(x)
        for u, v in zip(ra[:4], rb[:4]):
            np.testing.assert_array_equal(u, v)
    a.close(), b.close()
    e = gym_b200.B200Env("Pendulum-v1", device=0)
    e.reset(seed=0)
    _refused(lambda: e.step(np.zeros(1, np.float32)), r"B200Env\.step\(\)")
    _refused(lambda: e.reset(seed=0), r"B200Env\.reset\(\)")
    e.step(np.zeros(1, np.float32))
    e.close()
    s = ShardedVectorEnv("CartPole-v1", 64, gather=None, device=0)
    s.reset(seed=0)
    _refused(lambda: s.step(_torch().zeros(64, dtype=_torch().int64, device="cuda:0")), "ShardedVectorEnv")
    s.close()


def test_invalid_action_in_a_replay_is_reported_by_the_next_eager_call():
    from gym_b200 import error
    torch = _torch()
    env = _make("CartPole-v1", 512)
    env.reset(seed=0)
    act = torch.zeros(512, dtype=torch.int64, device="cuda:0")
    graph, _ = _capture(lambda: env.step(act))
    graph.replay()
    act[77] = 5
    graph.replay()
    torch.cuda.synchronize()
    with pytest.raises(error.InvalidAction):
        env.step(torch.zeros(512, dtype=torch.int64, device="cuda:0"))
    env.close()


@needs_reference
def test_gym_compat_vector_env_captures():
    ref_gym.import_reference()
    from gym_b200.gym_compat import GymVectorEnv
    a, b = GymVectorEnv("Acrobot-v1", 512, device=0), GymVectorEnv("Acrobot-v1", 512, device=0)
    a.reset(seed=3)
    b.reset(seed=3)
    a.action_space.seed(5)
    b.action_space.seed(5)
    _assert_same({"a": a.sample_actions()}, {"a": b.sample_actions()}, "eager draw")
    graph, out = _capture(lambda: _flat(a.step(a.sample_actions())))
    for k in range(20):
        graph.replay()
        _assert_same(out, _flat(b.step(b.sample_actions())), f"replay {k}")
    a.close(), b.close()
