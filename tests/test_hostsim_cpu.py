"""The DEVICE source of the step and reset kernels, compiled for the CPU, against the C oracle.  Runs without a GPU.

tests/hostsim/hostsim.cpp includes gym_b200/csrc/{rng,envs,b2lite,lunar,walker,per_env}.cuh and box2d_consts.h
through a small CUDA shim and calls the kernels' own per-env drivers (per_env.cuh) with plain loops, in the order the
kernels are launched.  What this pins on every CPU run: the drivers (action decode, TimeLimit, autoreset, final
observations, the Box2D step / TOI / reset passes with their parked-env and reset lists), the register-resident
solver (compile-time island topology), the scenes, the record packing (load_world / store_world), the host-computed
shape / mass / joint constants and the numpy-compatible RNG of the device code are bit-identical to the independent
C implementation in oracle/ -- the same statement tests/test_gpu_lunar.py / test_gpu_walker.py make on the GPU for
the nvcc build of this source.  (Not covered here: the kernels' thread and warp logic -- indexing, the
warp-synchronous TOI rounds, the shared-memory tiles of kernels P, B and G --, launch code and nvcc's code
generation -- that is what the `-m gpu` tests are for.)
"""
import numpy as np
import pytest

from hostsim import sim
from hostsim.sim import HostSim
from oracle import oracle as orc


def _compare(t, got, want, reward_atol=0.0):
    for k, name in enumerate(("obs", "reward", "terminated", "truncated")):
        if k == 1 and reward_atol:
            np.testing.assert_allclose(got[1], want[1], rtol=0, atol=reward_atol, err_msg=f"step {t}: reward")
            continue
        if not np.array_equal(got[k], want[k]):
            bad = np.argwhere(np.asarray(got[k]) != np.asarray(want[k]))
            raise AssertionError(f"step {t}: {name} differs at {bad[0]}: {np.asarray(got[k])[tuple(bad[0])]!r} "
                                 f"vs {np.asarray(want[k])[tuple(bad[0])]!r} ({len(bad)} values)")
    done = want[2] | want[3]
    assert np.array_equal(got[4][done], want[4][done]), f"step {t}: final observations"
    return done


LUNAR = [
    ("LunarLander", dict(), "random"),
    ("LunarLander", dict(), "heuristic"),
    ("LunarLanderContinuous", dict(), "random"),
    ("LunarLanderContinuous", dict(gravity=-6.5), "heuristic"),
    ("LunarLander", dict(enable_wind=True, wind_power=19.0, turbulence_power=1.9, gravity=-11.5), "random"),
    ("LunarLanderContinuous", dict(enable_wind=True), "heuristic"),
]


@pytest.mark.parametrize("name,kwargs,policy", LUNAR)
def test_lunar_device_source_on_cpu_equals_oracle(name, kwargs, policy):
    N, T, seed = 96, 400, 5
    cont = name.endswith("Continuous")
    rng = np.random.default_rng(2)
    extra = {}
    if kwargs.get("enable_wind"):
        extra = dict(wind_idx=rng.integers(-9999, 9999, size=N), torque_idx=rng.integers(-9999, 9999, size=N))
    sim = HostSim(name, N, 1000, **kwargs, **extra)
    ref = orc.OracleLunar(N, max_episode_steps=1000, continuous=cont, **kwargs, **extra)
    cur = ref.reset(seed=seed)
    assert np.array_equal(sim.reset(seed=seed), cur)
    n_done = n_sleep = 0
    for t in range(T):
        if policy == "random":
            a = rng.uniform(-1.6, 1.6, size=(N, 2)).astype(np.float32) if cont else rng.integers(0, 4, size=N)
        else:
            a = np.stack([orc.lunar_heuristic(s, continuous=cont) for s in cur])
        want = ref.step(a)
        done = _compare(t, sim.step(a), want)
        n_done += int(done.sum())
        n_sleep += int((want[1][want[2]] == 100).sum())
        cur = want[0]
    assert n_done > 0
    if policy == "heuristic" and not kwargs.get("enable_wind"):
        assert n_sleep > N // 3
    if kwargs.get("enable_wind"):
        assert all(np.array_equal(x, y) for x, y in zip(sim.wind_idx(), ref.wind_idx()))


@pytest.mark.parametrize("name,hardcore,policy", [("BipedalWalker", False, "gait"), ("BipedalWalkerHardcore", True, "gait"),
                                                  ("BipedalWalker", False, "random"), ("BipedalWalkerHardcore", True, "random")])
def test_walker_device_source_on_cpu_equals_oracle(name, hardcore, policy):
    N, T, seed = 24, 420, 31
    steps = 2000 if hardcore else 1600
    sim = HostSim(name, N, steps)
    ref = orc.OracleWalker(N, hardcore=hardcore, max_episode_steps=steps)
    cur = ref.reset(seed=seed)
    assert np.array_equal(sim.reset(seed=seed), cur)
    for i in range(N):
        t, boxes = sim.terrain(i)
        assert np.array_equal(t, ref.terrain(i)) and np.array_equal(boxes, ref.polys(i))
    rng = np.random.default_rng(8)
    gaits = [orc.WalkerHeuristic() for _ in range(N)]
    a = np.zeros((N, 4), dtype=np.float32)
    n_done = 0
    for t in range(T):
        if policy == "random":
            a = rng.uniform(-1.3, 1.3, size=(N, 4)).astype(np.float32)
        want = ref.step(a)
        done = _compare(t, sim.step(a), want)
        n_done += int(done.sum())
        if policy == "gait":
            for i in range(N):
                if done[i]:
                    gaits[i] = orc.WalkerHeuristic()
                    a[i] = 0.0
                else:
                    a[i] = gaits[i](want[0][i])
    assert n_done > (N // 2 if policy == "random" or hardcore else 0)


@pytest.mark.parametrize("defer", [True, False], ids=["deferred", "inline"])
@pytest.mark.parametrize("name", ["LunarLander", "BipedalWalkerHardcore"])
def test_box2d_step_configurations_on_cpu_equal_oracle(name, defer):
    """The Box2D step as the device can run it: with the TOI and reset passes deferred (the default) or inline in the
    step pass, and with the batch split into three launch ranges, the last one ragged, as the host path splits it
    into chunks.  Every configuration must give the oracle's trajectories bit for bit, and the deferred one must
    really have parked envs for the TOI pass and reset envs from the reset list."""
    lunar = name == "LunarLander"
    N, T, steps = (40, 160, 1000) if lunar else (20, 120, 2000)
    sim = HostSim(name, N, steps, defer=defer, ranges=3)
    ref = orc.OracleLunar(N, max_episode_steps=steps) if lunar else orc.OracleWalker(N, hardcore=True, max_episode_steps=steps)
    assert np.array_equal(sim.reset(seed=12), ref.reset(seed=12))
    rng = np.random.default_rng(6)
    n_done = 0
    for t in range(T):
        a = rng.integers(0, 4, size=N) if lunar else rng.uniform(-1.3, 1.3, size=(N, 4)).astype(np.float32)
        n_done += int(_compare(t, sim.step(a), ref.step(a)).sum())
    assert n_done > N // 2
    toi, reset = sim.list_totals()
    if defer:
        assert toi > 0 and reset == n_done, (toi, reset, n_done)
    else:
        assert toi == reset == 0


def test_manifold_table_overflow_is_handled_identically():
    """The Box2D scenes keep at most 8 (LunarLander) / 10 (BipedalWalker) touching pairs per env; real Box2D has no
    limit, and random play never gets there (max 7 observed), so the rule for a full table -- the extra pair counts
    as NOT touching: no constraint, no BeginContact, EndContact if it was touching -- cannot be tested at the shipped
    capacities.  Here both sides run with tiny tables (device source built with 1 / 2 slots, oracle told the same):
    overflows happen in most episodes, are counted on both sides, and the trajectories stay bit-identical."""
    from hostsim.sim import SMALLCAP
    try:
        orc.set_box2d_max_contacts(lunar=SMALLCAP["lunar"], walker=SMALLCAP["walker"])
        rng = np.random.default_rng(4)
        N, T = 64, 260
        sim = HostSim("LunarLander", N, 1000, smallcap=True)
        ref = orc.OracleLunar(N, max_episode_steps=1000)
        assert np.array_equal(sim.reset(seed=3), ref.reset(seed=3))
        for t in range(T):
            a = rng.integers(0, 4, size=N)
            _compare(t, sim.step(a), ref.step(a))
        assert sim.overflows() == ref.overflows() > 0
        sim.close()
        ref.close()
        N, T = 16, 200
        sim = HostSim("BipedalWalkerHardcore", N, 2000, smallcap=True)
        ref = orc.OracleWalker(N, hardcore=True, max_episode_steps=2000)
        assert np.array_equal(sim.reset(seed=9), ref.reset(seed=9))
        for t in range(T):
            a = rng.uniform(-1.0, 1.0, size=(N, 4)).astype(np.float32)
            _compare(t, sim.step(a), ref.step(a))
        assert sim.overflows() == ref.overflows() > 0
        sim.close()
        ref.close()
    finally:
        orc.set_box2d_max_contacts()
    # at the shipped capacities random play never overflows (this is what the GPU tests assert on the device too)
    ref = orc.OracleLunar(256, max_episode_steps=1000)
    ref.reset(seed=1)
    for t in range(300):
        ref.step(rng.integers(0, 4, size=256))
    assert ref.overflows() == 0
    ref.close()


# ---------------------------------------------------------------------------------------------------------
# classic control: gym_b200/csrc/envs.cuh on the CPU
# ---------------------------------------------------------------------------------------------------------
CLASSIC = [("CartPole-v1", 0, None), ("MountainCar-v0", 1, None), ("MountainCarContinuous-v0", 2, None),
           ("Pendulum-v1", 3, 10.0), ("Acrobot-v1", 4, None)]


@pytest.mark.parametrize("env_id,kind,param0", CLASSIC)
def test_classic_device_source_on_cpu_equals_oracle(env_id, kind, param0):
    """Same libm on both sides (glibc), so the only thing that may differ from the oracle is the transcription of
    the dynamics in envs.cuh -- and CartPole's own small-angle sin/cos kernel (csrc/envs.cuh: sincos_small), which
    replaces libm on the device and is within 1 ulp of it (next test)."""
    from hostsim.sim import HostSimClassic
    N, T, seed = 512, 600, 17
    ref = orc.OracleVec(env_id, N, max_episode_steps=150)       # several TimeLimit truncations within T steps
    sim = HostSimClassic(kind, N, 150, param0 or 0.0)
    assert np.array_equal(sim.reset(seed=seed), ref.reset(seed=seed))
    rng = np.random.default_rng(1)
    n_done = 0
    for t in range(T):
        if ref.act_dim == 0:
            a = rng.integers(0, ref.num_actions, size=N)
        else:
            a = rng.uniform(-2.5, 2.5, size=(N, 1)).astype(np.float32)
        want = ref.step(a)
        # Pendulum: the device squares the float32 torque as u*u where numpy calls powf(u, 2) (1 float32 ulp apart
        # for 0.08 % of inputs; DESIGN.md "Numerics"): rewards within 1e-9, everything else identical
        n_done += int(_compare(t, sim.step(a), want, reward_atol=1e-9 if kind == 3 else 0.0).sum())
    if kind == 0:   # CartPole: sincos_small is within 1 ulp of glibc, not identical; the float32 outputs above are
        np.testing.assert_allclose(sim.state(), ref.get_state()[0], rtol=1e-9, atol=1e-12)
    else:
        assert np.array_equal(sim.state(), ref.get_state()[0])
    assert n_done > N // 2


def test_cartpole_small_angle_sincos_against_libm():
    """csrc/envs.cuh: sincos_small (fdlibm's kernels without range reduction) against glibc over the angles CartPole
    is stepped at (|theta| <= 0.42 rad incl. the terminal step): never more than 1 ulp apart, identical for the
    overwhelming majority of inputs.  (The 1-ulp cases are why CartPole's float64 STATE is compared with a tolerance
    while every float32 output -- observations, rewards, flags -- is bit-identical.)"""
    import math
    from hostsim.sim import sincos_small
    rng = np.random.default_rng(0)
    x = np.concatenate([rng.uniform(-0.42, 0.42, 60000), rng.normal(0, 0.05, 60000).clip(-0.42, 0.42),
                        np.array([0.0, -0.0, 1e-300, -1e-300, 2.0 ** -27, 0.2094395102393195, 0.42, -0.42])])
    sn, cs = sincos_small(x)
    ws = np.array([math.sin(v) for v in x])
    wc = np.array([math.cos(v) for v in x])
    ulp_s = np.abs(sn.view(np.int64) - ws.view(np.int64))
    ulp_c = np.abs(cs.view(np.int64) - wc.view(np.int64))
    assert ulp_s.max() <= 1 and ulp_c.max() <= 1, (ulp_s.max(), ulp_c.max())
    assert (ulp_s == 0).mean() > 0.95 and (ulp_c == 0).mean() > 0.95, ((ulp_s == 0).mean(), (ulp_c == 0).mean())
    nz = x != 0
    assert np.array_equal(np.signbit(sn[nz]), np.signbit(ws[nz]))
    # sin(-0.0) comes out as +0.0 (libm: -0.0): only the sign of a zero product / zero sum downstream, never a value
    assert sn[x == 0].tolist() == [0.0, 0.0]


def test_restated_glibc_sin_cos_are_bit_identical_to_libm():
    """csrc/glibc_trig.cuh (glibc's sin / cos restated, FMA contractions included) against the libm of this very
    process -- the one the reference's math.sin / np.cos end in -- over the argument ranges the envs produce and far
    beyond: every result identical, bit for bit.  This is what lets Acrobot (chaotic: a 1-ulp difference grows by
    e^(0.09 t)) match the reference over whole free-running episodes."""
    import math
    from hostsim.sim import glibc_trig, glibc_trig_mismatches
    edge = np.array([0.0, -0.0, 2.0 ** -27, 2.0 ** -26, 1.4e-8, 0.126, -0.126, 0.12599999, 0.855469, 0.8554687, 0.85546875,
                     2.426265, 2.4262657, -2.426265, math.pi, -math.pi, math.pi / 2, 3 * math.pi / 2, 1e-300, 105414349.0,
                     0.5 * math.pi - 1e-9, 100 * math.pi, 12345.678, -7.0, 25.132741228718345])
    sn, cs = glibc_trig(edge)
    assert sn.tobytes() == np.array([math.sin(v) for v in edge]).tobytes()
    assert cs.tobytes() == np.array([math.cos(v) for v in edge]).tobytes()
    for k, (lo, hi) in enumerate([(-0.2, 0.2), (-1.0, 1.0), (-3.2, 3.2), (-10.0, 10.0), (-100.0, 100.0), (-1e6, 1e6),
                                  (-1.05e8, 1.05e8), (-1e-7, 1e-7)]):
        assert glibc_trig_mismatches(1000 + k, 2_000_000, lo, hi) == 0, (lo, hi)


def test_restated_glibc_square_is_bit_identical_to_libm_pow():
    """`x**2` in the reference is libm pow(x, 2.0), which is NOT x * x (1 ulp apart in ~0.09 % of arguments: enough to
    lose a chaotic Acrobot trajectory); csrc/glibc_trig.cuh: gt::sq restates glibc's pow for that exponent.  Against
    the libm of this process: identical everywhere."""
    from hostsim.sim import glibc_sq_mismatches
    total_neq = 0
    for k, (lo, hi) in enumerate([(-4.0, 4.0), (-30.0, 30.0), (0.9, 1.1), (-1e-3, 1e-3), (-1e6, 1e6), (1.0, 2.5)]):
        bad, neq = glibc_sq_mismatches(50 + k, 2_000_000, lo, hi)
        assert bad == 0, (lo, hi, bad)
        total_neq += neq
    assert total_neq > 1000     # the premise: pow(x, 2.0) really differs from x * x


def test_lunar_random_constructor_arguments_sweep():
    """Random LunarLander constructor arguments (gravity in (-12, 0), wind and turbulence powers, both action
    spaces, random wind phases): device source on the CPU == oracle."""
    rng = np.random.default_rng(123)
    for case in range(8):
        cont = bool(rng.integers(0, 2))
        wind = bool(rng.integers(0, 2))
        kw = dict(gravity=float(rng.uniform(-11.9, -0.5)))
        extra = {}
        if wind:
            kw.update(enable_wind=True, wind_power=float(rng.uniform(0, 20)), turbulence_power=float(rng.uniform(0, 2)))
            extra = dict(wind_idx=rng.integers(-9999, 9999, size=32), torque_idx=rng.integers(-9999, 9999, size=32))
        name = "LunarLanderContinuous" if cont else "LunarLander"
        sim = HostSim(name, 32, 120, **kw, **extra)
        ref = orc.OracleLunar(32, max_episode_steps=120, continuous=cont, **kw, **extra)
        seed = int(rng.integers(0, 2 ** 40))
        assert np.array_equal(sim.reset(seed=seed), ref.reset(seed=seed)), (case, kw)
        for t in range(150):
            a = rng.uniform(-1.2, 1.2, size=(32, 2)).astype(np.float32) if cont else rng.integers(0, 4, size=32)
            _compare(t, sim.step(a), ref.step(a))


import self_fixtures  # noqa: E402


@pytest.mark.parametrize("name", self_fixtures.names())
def test_device_source_on_cpu_reproduces_the_frozen_rollouts(name):
    d = self_fixtures.load(name)
    kw = dict(d["kwargs"])
    if d["family"] == "lunar":
        sim = HostSim("LunarLanderContinuous" if kw.pop("continuous", False) else "LunarLander", d["n"],
                      d["max_episode_steps"], **kw)
    else:
        sim = HostSim("BipedalWalkerHardcore" if kw.pop("hardcore", False) else "BipedalWalker", d["n"],
                      d["max_episode_steps"])
    self_fixtures.check(d, sim.step, sim.reset(seed=d["seed"]))


def test_toi_shortcuts_never_dismiss_a_pair_that_touches():
    """b2lite_toi.cuh skips b2TimeOfImpact when `toi_cannot_touch` proves that the pair's alpha is 1 (the polygon's
    box over its sweep stays beyond the touching distance of the fixture's box, or the whole polygon starts beyond a
    face line of the fixture by more than it can move).  The oracle applies no shortcut, so the bit-for-bit roll-outs
    above already check this; here the claim itself is fuzzed: 60 000 random sweeps of the task polygons near an
    edge / a box -- resting, sliding, rotating, approaching, tunnelling -- and whenever the shortcut fires the full
    b2TimeOfImpact of the same sweep must not report e_touching.  Both outcomes must occur often."""
    rng = np.random.default_rng(42)
    fired = touching = both = 0
    for k in range(60000):
        shape = int(rng.integers(0, 5))
        slope = rng.uniform(-0.6, 0.6)
        edge = ((-1.0, -slope), (1.0, slope))
        box = None
        if k % 4 == 3:
            edge, box = None, (-0.5, -1.0, 0.5, 0.0)
        mode = k % 3
        x0 = rng.uniform(-1.2, 1.2)
        h0 = abs(rng.normal(0.0, 0.6)) if mode else rng.uniform(0.0, 0.05)     # height of the body's centre region
        c0 = (x0, (slope * x0 if box is None else 0.0) + 0.6 * rng.uniform(0.2, 1.6) + h0)
        a0 = rng.uniform(-3.2, 3.2)
        if mode == 0:      # nearly at rest
            dc, da = rng.normal(0, 0.002, 2), rng.normal(0, 0.002)
        elif mode == 1:    # moderate motion
            dc, da = rng.normal(0, 0.08, 2), rng.normal(0, 0.08)
        else:              # fast, mostly downwards
            dc, da = np.array([rng.normal(0, 0.3), -abs(rng.normal(0, 1.0))]), rng.normal(0, 0.4)
        st, t, skip = sim.toi_probe(shape, c0, a0, (c0[0] + dc[0], c0[1] + dc[1]), a0 + da, edge=edge, box=box)
        fired += skip
        touching += st == 3
        both += skip and st == 3
    assert both == 0, f"{both} sweeps were dismissed although b2TimeOfImpact reports e_touching"
    assert fired > 5000 and touching > 5000, (fired, touching)



def test_device_time_of_impact_equals_the_oracles_on_random_sweeps():
    """`time_of_impact` / `gjk_distance` / the separation function of b2lite_toi.cuh (device source, compiled for the
    host) against oracle/b2lite_toi.h on the same 20 000 sweeps of the three task boxes whose body origin is the
    centre of mass (lander leg, walker upper / lower leg) against an edge: state and t bit for bit.  The roll-outs
    above cover this through whole episodes; this pins the function itself, fast spins and tunnelling included."""
    from oracle import oracle as orc
    polys = {}
    for shape in (1, 3, 4):
        verts, lc = sim.shape_verts(shape)
        assert len(verts) == 4 and not lc.any()
        polys[shape] = verts
    rng = np.random.default_rng(8)
    states = {}
    for k in range(20000):
        shape = (1, 3, 4)[k % 3]
        slope = rng.uniform(-0.6, 0.6)
        edge = ((-2.0, -2.0 * slope), (2.0, 2.0 * slope))
        x0 = rng.uniform(-1.0, 1.0)
        c0 = (x0, slope * x0 + rng.uniform(0.0, 1.2))
        a0 = rng.uniform(-3.2, 3.2)
        scale = (0.01, 0.1, 1.0)[(k // 3) % 3]
        c1 = (c0[0] + scale * rng.normal(0, 0.4), c0[1] - scale * abs(rng.normal(0, 1.0)))
        a1 = a0 + scale * rng.normal(0, 1.0)
        st, t, _ = sim.toi_probe(shape, c0, a0, c1, a1, edge=edge)
        ost, ot = orc.toi_probe(polys[shape], c0, a0, c1, a1, edge[0], edge[1])
        assert (st, np.float32(t).tobytes()) == (ost, np.float32(ot).tobytes()), (k, shape, st, t, ost, ot)
        states[st] = states.get(st, 0) + 1
    assert states.get(3, 0) > 3000 and states.get(4, 0) > 3000 and states.get(1, 0) == 0, states
