"""CPU tests of the Box2D-task oracles (oracle/lunar_oracle.c, oracle/walker_oracle.c).

PARITY UNPINNED for the rigid-body arithmetic (box2d-py is not installable here).  What can be pinned
on the CPU and is pinned here:
  * the reference's own behavioural test at this boundary (tests/envs/test_env_implementation.py:13-17:
    the heuristic controller scores > 100 on LunarLander-v2 at seed 1), discrete and continuous;
  * the numpy dtype flow (NEP 50) of the engine arithmetic in LunarLander.step (lunar_lander.py:479-554),
    checked against numpy scalars evaluating the same expressions;
  * the wind / gravity / continuous-action variants' documented semantics (lunar_lander.py:449-477,
    211-213, 480).
"""
import math

import numpy as np
import pytest

from oracle import oracle as orc


def _run_heuristic(env, continuous, seed, max_steps=1000):
    s = env.reset(seed=seed)[0]
    total, steps = 0.0, 0
    while True:
        a = orc.lunar_heuristic(s, continuous=continuous)
        obs, r, te, tr, fo = env.step(np.asarray([a]))
        total += float(r[0])
        steps += 1
        if te[0] or tr[0] or steps >= max_steps:
            return total, steps, bool(te[0])
        s = obs[0]


def test_reference_behavioural_test_heuristic_lands_discrete():
    total, steps, term = _run_heuristic(orc.OracleLunar(1), False, seed=1)
    assert term and total > 100, (total, steps)


def test_heuristic_lands_continuous():
    """demo_heuristic_lander with continuous=True (lunar_lander.py:766-768): same criterion."""
    total, steps, term = _run_heuristic(orc.OracleLunar(1, continuous=True), True, seed=1)
    assert term and total > 100, (total, steps)


@pytest.mark.parametrize("continuous", [False, True])
def test_heuristic_return_distribution_clears_the_reward_threshold(continuous):
    """Trajectory-level sanity of the re-derived physics (no real Box2D to compare with): the reference's heuristic
    controller (lunar_lander.py:683-763) is tuned on real Box2D and "solves" the task there, i.e. averages above the
    registry's reward_threshold of 200 (gym/envs/__init__.py:56-68).  On the oracle, seeds 0..99: discrete mean 238,
    median 266, 90 % of episodes above 200; continuous mean 280, 99 % above 200; every episode ends by termination
    (landed asleep or crashed), not by the 1000-step limit, bar one."""
    N = 100
    env = orc.OracleLunar(N, continuous=continuous)
    s = env.reset(seed=0)
    total, done, term = np.zeros(N), np.zeros(N, dtype=bool), np.zeros(N, dtype=bool)
    for _ in range(1000):
        a = np.asarray([orc.lunar_heuristic(s[i], continuous=continuous) for i in range(N)])
        s, r, te, tr, _fo = env.step(a)
        total += np.where(done, 0.0, r)
        term |= te & ~done
        done |= te | tr
        if done.all():
            break
    assert done.all() and term.mean() >= 0.98
    assert total.mean() > 200.0 and np.median(total) > 250.0, (total.mean(), np.median(total))
    assert (total > 200.0).mean() >= (0.95 if continuous else 0.85), (total > 200.0).mean()
    env.close()


def _numpy_engines(continuous, action, ang, posx, posy, disp0, disp1):
    """LunarLander.step's engine arithmetic (lunar_lander.py:479-554) evaluated by numpy/Python scalars with
    the types the reference has at each point: tip/side/dispersion/position are Python floats, the clipped
    continuous action is a float32 array.  Returns what Box2D receives (float32 pairs) + the fuel costs."""
    SCALE, MAIN, SIDE = 30.0, 13.0, 0.6
    if continuous:
        action = np.clip(action, -1, +1).astype(np.float32)
    tip = (math.sin(ang), math.cos(ang))
    side = (-tip[1], tip[0])
    dispersion = [disp0, disp1]
    out = np.zeros(8, dtype=np.float32)
    cost = [0.0, 0.0]
    on = [0, 0]
    m_power = 0.0
    if (continuous and action[0] > 0.0) or (not continuous and action == 2):
        m_power = (np.clip(action[0], 0.0, 1.0) + 1.0) * 0.5 if continuous else 1.0
        ox = tip[0] * (4 / SCALE + 2 * dispersion[0]) + side[0] * dispersion[1]
        oy = -tip[1] * (4 / SCALE + 2 * dispersion[0]) - side[1] * dispersion[1]
        impulse_pos = (posx + ox, posy + oy)
        out[0:4] = [-ox * MAIN * m_power, -oy * MAIN * m_power, impulse_pos[0], impulse_pos[1]]
        on[0] = 1
    s_power = 0.0
    if (continuous and np.abs(action[1]) > 0.5) or (not continuous and action in [1, 3]):
        if continuous:
            direction = np.sign(action[1])
            s_power = np.clip(np.abs(action[1]), 0.5, 1.0)
        else:
            direction = action - 2
            s_power = 1.0
        ox = tip[0] * dispersion[0] + side[0] * (3 * dispersion[1] + direction * 12.0 / SCALE)
        oy = -tip[1] * dispersion[0] - side[1] * (3 * dispersion[1] + direction * 12.0 / SCALE)
        impulse_pos = (posx + ox - tip[0] * 17 / SCALE, posy + oy + tip[1] * 14.0 / SCALE)
        out[4:8] = [-ox * SIDE * s_power, -oy * SIDE * s_power, impulse_pos[0], impulse_pos[1]]
        on[1] = 1
    reward = np.float64(0.0)
    r1 = reward - m_power * 0.30
    r2 = reward - s_power * 0.03
    cost = [float(-r1), float(-r2)]
    return out, np.asarray(cost), np.asarray(on)


@pytest.mark.parametrize("continuous", [False, True])
def test_engine_arithmetic_follows_numpy_dtype_flow(continuous):
    rng = np.random.default_rng(5)
    for k in range(4000):
        ang = float(np.float32(rng.uniform(-1.5, 1.5)))
        posx = float(np.float32(rng.uniform(0, 20)))
        posy = float(np.float32(rng.uniform(0, 14)))
        d0, d1 = rng.uniform(-1.0, 1.0) / 30.0, rng.uniform(-1.0, 1.0) / 30.0
        if continuous:
            action = rng.uniform(-1.5, 1.5, size=2).astype(np.float32)
            if k % 17 == 0:
                action[1] = np.float32(0.5)      # boundary of the side-engine dead zone
            if k % 19 == 0:
                action[0] = np.float32(0.0)
        else:
            action = int(rng.integers(0, 4))
        want, wcost, won = _numpy_engines(continuous, action, ang, posx, posy, d0, d1)
        got, gcost, gon = orc.lunar_engines(continuous, action, ang, posx, posy, d0, d1)
        assert np.array_equal(won, gon), (k, action)
        assert np.array_equal(want.view(np.uint32), got.view(np.uint32)), (k, action, want, got)
        assert np.array_equal(wcost, gcost), (k, action, wcost, gcost)


def test_continuous_actions_are_clipped_and_dead_zones_hold():
    """lunar_lander.py:152-160,480: main engine off for a0 <= 0, side engines off for |a1| <= 0.5; values
    beyond +-1 behave as +-1."""
    def roll(a, steps=30):
        e = orc.OracleLunar(1, continuous=True)
        e.reset(seed=3)
        out = []
        for _ in range(steps):
            out.append(e.step(np.asarray([a], dtype=np.float32))[0][0].copy())
        return np.stack(out)
    assert np.array_equal(roll([0.0, 0.0]), roll([-0.7, 0.5]))      # both dead zones
    assert np.array_equal(roll([1.0, 1.0]), roll([3.0, 7.0]))       # clipped
    assert not np.array_equal(roll([0.0, 0.0]), roll([0.01, 0.0]))  # main engine fires at 50 % from a0 > 0
    assert not np.array_equal(roll([0.0, 0.0]), roll([0.0, -0.51]))
    # discrete action 0 == continuous [0, 0]; discrete 2 == continuous [1, 0] (m_power 1.0)
    d = orc.OracleLunar(1)
    d.reset(seed=3)
    dn = np.stack([d.step(np.asarray([0]))[0][0].copy() for _ in range(30)])
    assert np.array_equal(dn, roll([0.0, 0.0]))


def test_gravity_parameter_sets_free_fall():
    """lunar_lander.py:211-213,240: world gravity (0, gravity).  One free-fall step changes v_y by g*dt."""
    dv = {}
    for g in (-10.0, -3.5, -11.9):
        e = orc.OracleLunar(1, gravity=g)
        e.reset(seed=0)
        v0 = e.bodies(0)[0][0, 4]
        e.step(np.asarray([0]))
        dv[g] = float(e.bodies(0)[0][0, 4] - v0)
        # the legs hang on motorised joints, so the lander's own dv is g*dt only up to their (g-independent) pull
        assert abs(dv[g] - g / 50.0) < 0.02, (g, dv[g])
    assert abs((dv[-10.0] - dv[-3.5]) - (-6.5 / 50.0)) < 1e-3, dv
    assert abs((dv[-11.9] - dv[-10.0]) - (-1.9 / 50.0)) < 1e-3, dv
    a = orc.OracleLunar(1, gravity=-10.0)
    b = orc.OracleLunar(1)
    assert np.array_equal(a.reset(seed=4), b.reset(seed=4))


def test_wind_semantics():
    """lunar_lander.py:449-477: wind only while neither leg touches; wind_idx/torque_idx advance by one per windy
    step, are per-object (drawn in __init__, :234-235) and survive reset()."""
    wi0, ti0 = 1234, -4321
    e = orc.OracleLunar(2, enable_wind=True, wind_idx=[wi0, wi0 + 7], torque_idx=[ti0, ti0])
    calm = orc.OracleLunar(2)
    o1 = e.reset(seed=9)
    o0 = calm.reset(seed=9)
    assert not np.array_equal(o1, o0)                     # the embedded step(0) of reset() already feels the wind
    wi, ti = e.wind_idx()
    assert wi.tolist() == [wi0 + 1, wi0 + 8] and ti.tolist() == [ti0 + 1, ti0 + 1]
    resets = 0
    for t in range(400):
        obs, r, te, trn, fo = e.step(np.asarray([0, 0]))
        wi2, ti2 = e.wind_idx()
        d = (wi2 - wi)
        assert set(d.tolist()) <= {0, 1, 2}                # 2: a windy step + the embedded step of an autoreset
        assert np.array_equal(wi2 - wi, ti2 - ti)
        resets += int((te | trn).sum())
        wi, ti = wi2, ti2
    assert resets >= 1                                     # crashed at least once: indices kept counting across reset
    assert (wi > np.asarray([wi0, wi0 + 7]) + 50).all()
    # zero wind power / zero turbulence == no wind at all (forces of exactly 0.0 are added)
    z = orc.OracleLunar(1, enable_wind=True, wind_power=0.0, turbulence_power=0.0, wind_idx=[5], torque_idx=[6])
    c = orc.OracleLunar(1)
    assert np.array_equal(z.reset(seed=2), c.reset(seed=2))
    for _ in range(50):
        assert np.array_equal(z.step(np.asarray([2]))[0], c.step(np.asarray([2]))[0])


def test_wind_stops_while_a_leg_touches_the_ground():
    e = orc.OracleLunar(1, enable_wind=True, wind_idx=[100], torque_idx=[200], wind_power=2.0, turbulence_power=0.1)
    s = e.reset(seed=1)[0]
    stalled = 0
    for _ in range(600):
        wi = e.wind_idx()[0][0]
        legs = bool(s[6] or s[7])
        obs, r, te, trn, fo = e.step(np.asarray([orc.lunar_heuristic(s)]))
        if te[0] or trn[0]:
            break
        d = e.wind_idx()[0][0] - wi
        assert d == (0 if legs else 1)
        stalled += legs
        s = obs[0]
    assert stalled > 0


def test_lunar_oracle_is_deterministic_and_seed_fanout_is_seed_plus_index():
    a = orc.OracleLunar(4)
    b = orc.OracleLunar(1)
    oa = a.reset(seed=10)
    ob = b.reset(seed=12)
    assert np.array_equal(oa[2], ob[0])
    rng = np.random.default_rng(0)
    for _ in range(150):
        act = rng.integers(0, 4, size=4)
        oa = a.step(act)[0]
        ob = b.step(act[2:3])[0]
        assert np.array_equal(oa[2], ob[0])


@pytest.mark.parametrize("kind", ["lunar", "walker"])
def test_oracle_window_stands_in_for_a_slice_of_the_batch(kind):
    """reset(seed, first=lo) of an m-env oracle seeds env k with seed + lo + k: it then steps exactly as envs
    [lo, lo + m) of a larger batch (how the GPU tests check windows of batches too large for the oracle)."""
    make = orc.OracleLunar if kind == "lunar" else orc.OracleWalker
    big, win = make(24), make(8)
    assert np.array_equal(big.reset(seed=7)[16:], win.reset(seed=7, first=16))
    rng = np.random.default_rng(1)
    for _ in range(40):
        act = rng.integers(0, 4, size=24) if kind == "lunar" else rng.uniform(-1, 1, size=(24, 4)).astype(np.float32)
        for x, y in zip(big.step(act), win.step(act[16:])):
            assert np.array_equal(x[16:], y)
    big.close()
    win.close()


def test_walker_oracle_invariants():
    """bipedal_walker.py:517-606: obs shape/dtype, lidar fractions in [0, 1], leg contact flags binary, reward
    -100 exactly on termination, truncation only from the TimeLimit."""
    e = orc.OracleWalker(8, max_episode_steps=300)
    o = e.reset(seed=0)
    assert o.shape == (8, 24) and o.dtype == np.float32
    rng = np.random.default_rng(1)
    saw_term = False
    for t in range(320):
        o, r, te, tr, fo = e.step(rng.uniform(-1, 1, size=(8, 4)).astype(np.float32))
        assert np.isfinite(o).all() and np.isfinite(r).all()
        assert ((o[:, 14:] >= 0) & (o[:, 14:] <= 1)).all()
        assert np.isin(o[:, 8], (0.0, 1.0)).all() and np.isin(o[:, 13], (0.0, 1.0)).all()
        assert (r[te] == -100).all()
        saw_term |= bool(te.any())
    assert saw_term


# ---------------------------------------------------------------------------------------------------------
# BipedalWalker / BipedalWalkerHardcore
# ---------------------------------------------------------------------------------------------------------
def _numpy_terrain(seed, hardcore, g=None):
    """BipedalWalker._generate_terrain (bipedal_walker.py:277-402) driven by a real numpy Generator: returns the
    200 terrain heights and the obstacle boxes (x0, ylo, x1, yhi) as float32, in creation order."""
    if g is None:
        g = np.random.Generator(np.random.PCG64(np.random.SeedSequence(seed)))
    SCALE = 30.0
    STEP, LENGTH, HEIGHT, GRASS_LEN, STARTPAD = 14 / SCALE, 200, 400 / SCALE / 4, 10, 20
    GRASS, STUMP, STAIRS, PIT, STATES = range(5)
    state, velocity, y, counter, oneshot = GRASS, 0.0, HEIGHT, STARTPAD, False
    ys, boxes = [], []
    steps = width = height = 0
    original_y = 0
    for i in range(LENGTH):
        x = i * STEP
        if state == GRASS and not oneshot:
            velocity = 0.8 * velocity + 0.01 * np.sign(HEIGHT - y)
            if i > STARTPAD:
                velocity += g.uniform(-1, 1) / SCALE
            y += velocity
        elif state == PIT and oneshot:
            counter = g.integers(3, 5)
            boxes.append((x, y - 4 * STEP, x + STEP, y))
            boxes.append((x + STEP * counter, y - 4 * STEP, x + STEP + STEP * counter, y))
            counter += 2
            original_y = y
        elif state == PIT and not oneshot:
            y = original_y
            if counter > 1:
                y -= 4 * STEP
        elif state == STUMP and oneshot:
            counter = g.integers(1, 3)
            boxes.append((x, y, x + counter * STEP, y + counter * STEP))
        elif state == STAIRS and oneshot:
            height = +1 if g.random() > 0.5 else -1
            width = g.integers(4, 5)
            steps = g.integers(3, 5)
            original_y = y
            for s in range(steps):
                boxes.append((x + (s * width) * STEP, y + (-1 + s * height) * STEP,
                              x + ((1 + s) * width) * STEP, y + (s * height) * STEP))
            counter = steps * width
        elif state == STAIRS and not oneshot:
            s = steps * width - counter - height
            n = s / width
            y = original_y + (n * height) * STEP
        oneshot = False
        ys.append(y)
        counter -= 1
        if counter == 0:
            counter = g.integers(GRASS_LEN / 2, GRASS_LEN)
            if state == GRASS and hardcore:
                state = g.integers(1, STATES)
            else:
                state = GRASS
            oneshot = True
    return np.asarray(ys, dtype=np.float32), np.asarray(boxes, dtype=np.float32).reshape(-1, 4)


@pytest.mark.parametrize("hardcore", [False, True])
def test_walker_terrain_is_pinned_to_numpy(hardcore):
    n = 24
    e = orc.OracleWalker(n, hardcore=hardcore)
    e.reset(seed=100)
    kinds = set()
    for i in range(n):
        ys, boxes = _numpy_terrain(100 + i, hardcore)
        assert np.array_equal(e.terrain(i).view(np.uint32), ys.view(np.uint32)), i
        got = e.polys(i)
        assert got.shape == boxes.shape and np.array_equal(got.view(np.uint32), boxes.view(np.uint32)), i
        assert len(boxes) <= 39
        if hardcore:
            assert len(boxes) >= 10
            w = np.round((boxes[:, 2] - boxes[:, 0]) / (14 / 30.0)).astype(int)
            kinds |= set(w.tolist())
        else:
            assert len(boxes) == 0
    if hardcore:
        assert {1, 2, 4} <= kinds          # pit walls / small stumps (1), big stumps (2), stair steps (4)


def _walk(hardcore, seed, max_steps):
    e = orc.OracleWalker(1, hardcore=hardcore, max_episode_steps=max_steps)
    s = e.reset(seed=seed)[0]
    gait = orc.WalkerHeuristic()
    a = np.zeros(4)
    total, track = 0.0, []
    for t in range(max_steps):
        obs, r, te, tr, fo = e.step(a.astype(np.float32)[None])
        total += float(r[0])
        if te[0] or tr[0]:
            return total, t + 1, bool(te[0]), float(r[0]), track, e
        track.append((e.bodies(0)[0].copy(), obs[0].copy()))
        a = gait(obs[0])
    return total, max_steps, False, 0.0, track, e


def test_walker_demo_gait_walks_the_course():
    """The reference's own demo controller (bipedal_walker.py:775-854) on the re-derived physics: it has to carry
    the walker over most of the 200-segment course (reward_threshold of the task is 300, gym/envs/__init__.py:74)."""
    totals = [_walk(False, seed, 1600)[0] for seed in (4, 5, 6)]   # 24 of the seeds 0..29 walk the whole course
    assert min(totals) > 300, totals


def test_hardcore_obstacles_are_solid_and_seen_by_the_lidar():
    stopped = 0
    for seed in range(4):
        total, steps, term, last_r, track, e = _walk(True, seed, 2000)
        assert term and last_r == -100.0           # the demo gait cannot pass the obstacles: it falls at one
        stopped += 1
    assert stopped == 4
    # geometry: replay seed 0 and look at the lower legs' corners against the obstacle boxes
    e = orc.OracleWalker(1, hardcore=True, max_episode_steps=2000)
    s = e.reset(seed=0)[0]
    boxes = e.polys(0)
    gait = orc.WalkerHeuristic()
    a = np.zeros(4)
    hx, hy = 0.8 * (8 / 30.0) / 2, (34 / 30.0) / 2
    corners = np.array([[-hx, -hy], [hx, -hy], [hx, hy], [-hx, hy]])
    deepest, min_lidar, reached = 0.0, 1.0, False
    for t in range(2000):
        obs, r, te, tr, fo = e.step(a.astype(np.float32)[None])
        if te[0] or tr[0]:
            break
        bodies = e.bodies(0)[0]
        for b in (2, 4):
            cx, cy, ang = bodies[b, 0], bodies[b, 1], bodies[b, 2]
            R = np.array([[np.cos(ang), -np.sin(ang)], [np.sin(ang), np.cos(ang)]])
            pts = corners @ R.T + np.array([cx, cy])
            for (x0, ylo, x1, yhi) in boxes:
                inside = (pts[:, 0] > x0) & (pts[:, 0] < x1) & (pts[:, 1] > ylo) & (pts[:, 1] < yhi)
                if inside.any():
                    d = np.minimum.reduce([pts[inside, 0] - x0, x1 - pts[inside, 0], pts[inside, 1] - ylo, yhi - pts[inside, 1]])
                    deepest = max(deepest, float(d.max()))
        reached |= bool(bodies[0, 0] + 1.5 > boxes[0, 0])
        min_lidar = min(min_lidar, float(obs[0, 14:].min()))
        a = gait(obs[0])
    assert reached                                   # the walker got to the first obstacle
    # ... and never sank into a box by more than one step of a ~6 m/s impact (no continuous collision in this
    # restatement; resting contacts stay within the solver's 0.005 slop + 0.01 skin)
    assert deepest < 0.15, deepest
    assert min_lidar < 0.35


# ---------------------------------------------------------------------------------------------------------
# physics invariants of the re-derived solver (independent of any Box2D implementation detail)
# ---------------------------------------------------------------------------------------------------------
def _poly_area(pts):
    x, y = np.asarray(pts, dtype=np.float64).T
    return 0.5 * abs(np.dot(x, np.roll(y, -1)) - np.dot(y, np.roll(x, -1)))


def _lunar_masses():
    """density x area of the fixtures of lunar_lander.py:354-368,379-398 (lander density 5, legs density 1)."""
    S = 30.0
    lander = _poly_area([(-14 / S, 17 / S), (-17 / S, 0), (-17 / S, -10 / S), (17 / S, -10 / S), (17 / S, 0), (14 / S, 17 / S)])
    leg = (2 * 2 / S) * (2 * 8 / S)
    return np.array([5.0 * lander, 1.0 * leg, 1.0 * leg])


def test_free_flight_conserves_momentum_up_to_gravity():
    """Joint impulses are internal: in free flight the linear momentum of lander + legs changes by exactly
    M g dt per step and nothing else (no engines: action 0; no wind)."""
    m = _lunar_masses()
    M = m.sum()
    for g in (-10.0, -4.0):
        e = orc.OracleLunar(1, gravity=g)
        e.reset(seed=6)
        b0 = e.bodies(0)[0].astype(np.float64)
        px0, py0 = float(m @ b0[:, 3]), float(m @ b0[:, 4])
        for k in range(1, 26):
            o = e.step(np.asarray([0]))[0][0]
            assert o[6] == 0 and o[7] == 0, "still in the air"
            b = e.bodies(0)[0].astype(np.float64)
            px, py = float(m @ b[:, 3]), float(m @ b[:, 4])
            assert abs(px - px0) < 2e-3 * M, (k, px - px0)                        # float32 solver round-off only
            assert abs((py - py0) - M * g * k / 50.0) < 2e-3 * M, (k, py - py0, M * g * k / 50.0)


def test_leg_joints_respect_their_limits_and_anchors():
    """The revolute joints hold: leg angles stay within [lower, upper] up to the solver's angular slop + one step of
    motion, and each leg's anchor keeps its distance to the lander's centre (the lander-side anchor is a fixed point
    of the lander) up to the linear slop, over a whole heuristic episode including the landing impacts."""
    e = orc.OracleLunar(1)
    s = e.reset(seed=1)[0]
    S = 30.0
    worst_angle = worst_anchor = 0.0
    d0 = {}
    for t in range(600):
        obs, r, te, tr, fo = e.step(np.asarray([orc.lunar_heuristic(s)]))
        if te[0] or tr[0]:
            break
        b = e.bodies(0)[0].astype(np.float64)
        for li, i in ((1, -1), (2, +1)):
            rel = b[li, 2] - b[0, 2]
            lo, hi = (0.4, 0.9) if i == -1 else (-0.9, -0.4)          # lunar_lander.py:405-412
            worst_angle = max(worst_angle, lo - rel, rel - hi)
            ca, sa = np.cos(b[li, 2]), np.sin(b[li, 2])
            ax, ay = i * 20 / S, 18 / S                               # localAnchorB, :402-404
            anchor = np.array([b[li, 0] + ca * ax - sa * ay, b[li, 1] + sa * ax + ca * ay])
            d = float(np.hypot(*(anchor - b[0, :2])))
            worst_anchor = max(worst_anchor, abs(d - d0.setdefault(li, d)))
        s = obs[0]
    assert t > 100
    assert worst_angle < 0.08, worst_angle          # 2 deg slop + impacts (the limit is soft within one step)
    assert worst_anchor < 0.02, worst_anchor


def test_landed_lander_comes_to_rest_and_sleeps():
    """A lander that has landed ends its episode through `not self.lander.awake` (+100, lunar_lander.py:594-596):
    the island has to fall below the sleep tolerances for 0.5 s while resting on two leg contacts."""
    e = orc.OracleLunar(1)
    s = e.reset(seed=1)[0]
    last = None
    for t in range(1000):
        obs, r, te, tr, fo = e.step(np.asarray([orc.lunar_heuristic(s)]))
        if te[0] or tr[0]:
            last = (float(r[0]), fo[0].copy())
            break
        s = obs[0]
    assert last is not None and last[0] == 100.0
    final = last[1]
    assert final[6] == 1.0 and final[7] == 1.0                      # both legs on the ground
    assert abs(final[2]) < 0.01 and abs(final[3]) < 0.01 and abs(final[5]) < 0.01
    assert abs(final[0]) < 0.3 and abs(final[4]) < 0.2               # on the pad, upright


# ---------------------------------------------------------------------------------------------------------
# continuous collision (b2World::SolveTOI, oracle/b2lite_toi.h)
# ---------------------------------------------------------------------------------------------------------
def test_time_of_impact_of_a_falling_box_matches_the_analytic_answer():
    """b2TimeOfImpact stops the core shapes at the target separation b2_linearSlop (0.005) +- a quarter of it.  A box of
    half-height 0.5 whose centre falls from y = 2 to y = -2 over the step, against the edge y = 0: the bottom face
    is at 1.5 - 4 t, so t = (1.5 - 0.005) / 4; same with a quarter turn of rotation (the lowest corner decides)."""
    box = [(-1.0, -0.5), (1.0, -0.5), (1.0, 0.5), (-1.0, 0.5)]
    st, t = orc.toi_probe(box, (0.0, 2.0), 0.0, (0.0, -2.0), 0.0, (-5.0, 0.0), (5.0, 0.0))
    assert st == 3 and abs((1.5 - 4 * t) - 0.005) <= 0.25 * 0.005 + 1e-6
    # far above the edge at the end of the step: separated, t = tMax
    st, t = orc.toi_probe(box, (0.0, 5.0), 0.0, (0.0, 3.0), 0.0, (-5.0, 0.0), (5.0, 0.0))
    assert (st, t) == (4, 1.0)
    # already closer than the target at t = 0: touching at t = 0
    st, t = orc.toi_probe(box, (0.0, 0.504), 0.0, (0.0, -1.0), 0.0, (-5.0, 0.0), (5.0, 0.0))
    assert (st, t) == (3, 0.0)
    # translating + rotating by 90 degrees: at the reported time the lowest corner is at the target height
    st, t = orc.toi_probe(box, (0.0, 3.0), 0.0, (0.0, -1.0), np.pi / 2, (-5.0, 0.0), (5.0, 0.0))
    assert st == 3 and 0.0 < t < 1.0
    ang, cy = t * np.pi / 2, 3.0 - 4.0 * t
    low = min(cy + np.sin(ang) * x + np.cos(ang) * y for x, y in box)
    assert abs(low - 0.005) <= 0.25 * 0.005 + 1e-5
    # moving along the edge without approaching it: separated
    st, t = orc.toi_probe(box, (-2.0, 1.0), 0.0, (2.0, 1.0), 0.0, (-5.0, 0.0), (5.0, 0.0))
    assert st == 4


def test_gjk_distance_matches_brute_force_geometry():
    """b2Distance as restated in oracle/b2lite_toi.h (simplex cache, Solve2 / Solve3, support mapping, duplicate-vertex
    termination) against an independent computation: the distance between a convex polygon and a segment is the
    minimum over (polygon vertex, segment) and (segment endpoint, polygon edge) point-to-segment distances when they
    do not overlap, and 0 when they do.  3 000 random poses of the lander's hexagon and of a thin leg box."""
    def seg_dist(p, a, b):
        ab, ap = b - a, p - a
        t = np.clip(np.dot(ap, ab) / np.dot(ab, ab), 0.0, 1.0)
        return float(np.linalg.norm(ap - t * ab))

    def intersects(p1, p2, q1, q2):
        def orient(a, b, c):
            return (b[0] - a[0]) * (c[1] - a[1]) - (b[1] - a[1]) * (c[0] - a[0])
        return (orient(p1, p2, q1) * orient(p1, p2, q2) < 0) and (orient(q1, q2, p1) * orient(q1, q2, p2) < 0)

    def inside(poly, p):
        n = len(poly)
        return all(((poly[(i + 1) % n][0] - poly[i][0]) * (p[1] - poly[i][1]) - (poly[(i + 1) % n][1] - poly[i][1]) * (p[0] - poly[i][0])) >= 0
                   for i in range(n))

    # both counter-clockwise, as b2PolygonShape::Set leaves them
    hexagon = np.array([(-17, -10), (17, -10), (17, 0), (14, 17), (-14, 17), (-17, 0)], dtype=np.float64) / 30.0
    leg = np.array([(-1, -4), (1, -4), (1, 4), (-1, 4)], dtype=np.float64) / 15.0
    rng = np.random.default_rng(5)
    checked = overlapping = 0
    for k in range(3000):
        poly = hexagon if k % 2 == 0 else leg
        a = rng.uniform(-3.2, 3.2)
        c = rng.uniform(-2.0, 2.0, 2)
        v1, v2 = rng.uniform(-2.0, 2.0, 2), rng.uniform(-2.0, 2.0, 2)
        if np.linalg.norm(v2 - v1) < 0.2:
            continue
        R = np.array([[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]])
        world = poly @ R.T + c
        n = len(world)
        overlap = inside(world, v1) or inside(world, v2) or any(intersects(world[i], world[(i + 1) % n], v1, v2) for i in range(n))
        want = 0.0 if overlap else min(min(seg_dist(p, v1, v2) for p in world),
                                       min(seg_dist(q, world[i], world[(i + 1) % n]) for q in (v1, v2) for i in range(n)))
        got, cnt = orc.distance_probe(poly, c, a, v1, v2)
        if overlap:
            overlapping += 1
            assert got < 1e-3 and cnt == 3 or got < 1e-4, (k, got, cnt)
        else:
            assert abs(got - want) <= 2e-5 + 2e-5 * want, (k, got, want, cnt)
            assert cnt in (1, 2)
        checked += 1
    assert checked > 2500 and overlapping > 100


def test_time_of_impact_lands_on_the_target_separation_and_not_later_than_first_contact():
    """b2TimeOfImpact's contract (b2TimeOfImpact.cpp: conservative advancement to `target` = max(linearSlop,
    totalRadius - 3 linearSlop) within 0.25 linearSlop), checked with the GJK distance that the test above ties to plain
    geometry: when the state is e_touching at t, the core shapes at the pose interpolated to t are `target` apart; when
    it is e_separated they are further apart than that at the end of the sweep.  For sweeps without rotation the
    separation along the fixed axis is linear in t, so the stronger statements hold too and are checked: no sampled
    earlier time is closer than `target`, and a separated sweep never comes closer anywhere.  (With rotation the
    algorithm itself can miss a shape that swings in and out within one step -- it only looks at the end of the
    interval along the current axis, "Is the final configuration separated?" -- and so does the restatement; case 1688
    of this generator with a spin of 1.24 rad is one.)  4 000 random sweeps of the lander's hexagon and a leg box."""
    slop = 0.005
    target, tol = max(slop, 4 * slop - 3 * slop), 0.25 * slop
    hexagon = np.array([(-17, -10), (17, -10), (17, 0), (14, 17), (-14, 17), (-17, 0)], dtype=np.float64) / 30.0
    leg = np.array([(-1, -4), (1, -4), (1, 4), (-1, 4)], dtype=np.float64) / 15.0
    rng = np.random.default_rng(11)
    eps = 2e-5
    n_touch = n_sep = n_other = n_start = 0
    for k in range(4000):
        poly = hexagon if k % 2 == 0 else leg
        slope = rng.uniform(-0.5, 0.5)
        v1, v2 = (-3.0, -3.0 * slope), (3.0, 3.0 * slope)
        x0 = rng.uniform(-1.0, 1.0)
        c0 = np.array([x0, slope * x0 + rng.uniform(0.7, 1.6)])
        a0 = rng.uniform(-3.0, 3.0)
        c1 = c0 + np.array([rng.normal(0, 0.4), -abs(rng.normal(0, 1.2))])
        spin = rng.normal(0, 0.5)
        translating = k % 4 < 2
        a1 = a0 if translating else a0 + spin
        st, t = orc.toi_probe(poly, c0, a0, c1, a1, v1, v2)
        pose = lambda b: ((1 - b) * c0 + b * c1, (1 - b) * a0 + b * a1)
        dist = lambda b: orc.distance_probe(poly, *pose(np.float32(b)), v1, v2)[0]
        if st == 3:
            n_touch += 1
            d = dist(t)
            if t == 0.0:       # already within reach at the start of the sweep
                assert 0.0 < d <= target + tol + eps, (k, d)
                n_start += 1
                continue
            assert target - tol - eps <= d <= target + tol + eps, (k, t, d)
            for b in np.linspace(0.0, t, 12, endpoint=False) if translating else ():
                assert dist(b) >= target - tol - eps, (k, t, b, dist(b))
        elif st == 4:
            n_sep += 1
            assert t == 1.0
            for b in np.linspace(0.0, 1.0, 16) if translating else (1.0,):
                assert dist(b) >= target - tol - eps, (k, b, dist(b))
        elif st == 2:      # e_overlapped: the cores already intersect at the start
            assert t == 0.0 and dist(0.0) == 0.0, (k, t, dist(0.0))
        else:
            n_other += 1
    assert n_touch - n_start > 800 and n_sep > 800 and n_other == 0, (n_touch, n_start, n_sep, n_other)


def test_toi_keeps_a_fast_lander_from_tunnelling_through_the_pad():
    """The lander thrown down at 95 m/s covers 1.9 m per step, more than its own height: the discrete solver alone
    lets it pass through the helipad (a thin edge has no inside) and it ends on the base edge at y = 0; with
    SolveTOI it is stopped on the pad (y = H/4 = 3.33) in the step in which it would have crossed it, and the
    contact listener ends the episode there.  lunar_lander.py:556,591-596; Box2D b2World::SolveTOI."""
    def drop(toi):
        orc.set_box2d_toi(toi)
        try:
            e = orc.OracleLunar(1)
            e.reset(seed=3)
            for b in range(3):
                e.set_body_velocity(0, b, 0.0, -95.0)
            ys = []
            for t in range(30):
                obs, r, te, tr, fo = e.step(np.zeros(1, dtype=np.int64))
                if te[0]:
                    return min(ys + [float((fo[0, 1]) * (400 / 30.0 / 2) + (400 / 30.0 / 4 + 18 / 30.0))]), float(r[0]), e.toi_stats()
                ys.append(float(e.bodies(0)[0][0, 1]))
            raise AssertionError("the lander never hit anything")
        finally:
            orc.set_box2d_toi(True)
    pad = 400 / 30.0 / 4
    low_off, r_off, (calls_off, ev_off) = drop(False)
    low_on, r_on, (calls_on, ev_on) = drop(True)
    assert r_off == -100.0 and r_on == -100.0
    assert ev_off == 0 and low_off < pad - 1.0          # went through the pad
    assert ev_on >= 1 and low_on > pad - 0.2            # stopped on it


def test_random_play_exercises_toi_sub_steps():
    """The bit-for-bit comparisons of the device source with this oracle (tests/test_hostsim_cpu.py, the -m gpu tests)
    run random / heuristic / gait play: make sure that play does go through TOI sub-steps, i.e. that those tests cover
    b2lite_toi as well, and that the candidate / manifold tables never overflow."""
    e = orc.OracleLunar(64)
    e.reset(seed=5)
    rng = np.random.default_rng(0)
    for t in range(300):
        e.step(rng.integers(0, 4, size=64))
    calls, events = e.toi_stats()
    assert events > 100 and calls > events and e.overflows() == 0
    w = orc.OracleWalker(16)
    w.reset(seed=5)
    for t in range(200):
        w.step(rng.uniform(-1, 1, (16, 4)).astype(np.float32))
    calls, events = w.toi_stats()
    assert events > 20 and calls > events and w.overflows() == 0


# ---------------------------------------------------------------------------------------------------------
# frozen roll-outs (tests/golden_self): the re-derived physics must not move between rounds
# ---------------------------------------------------------------------------------------------------------
import self_fixtures  # noqa: E402


@pytest.mark.parametrize("name", self_fixtures.names())
def test_oracle_reproduces_its_frozen_rollouts(name):
    d = self_fixtures.load(name)
    kw = dict(d["kwargs"])
    if d["family"] == "lunar":
        env = orc.OracleLunar(d["n"], max_episode_steps=d["max_episode_steps"], **kw)
    else:
        env = orc.OracleWalker(d["n"], max_episode_steps=d["max_episode_steps"], **kw)
    self_fixtures.check(d, env.step, env.reset(seed=d["seed"]))


def test_frozen_rollouts_cover_the_interesting_events():
    ds = {n: self_fixtures.load(n) for n in self_fixtures.names()}
    assert len(ds) >= 7
    lh = ds["lunarlander_v2_heuristic"]
    first_done = int(np.argmax(lh["terminated"][:, 0]))
    assert abs(float(lh["reward"][:first_done + 1, 0].sum()) - 262.03) < 0.01     # the seed-1 landing of DESIGN.md
    assert (lh["reward"][lh["terminated"]] == 100).all()                          # every episode ends asleep on the pad
    assert (ds["lunarlander_v2_random"]["reward"][ds["lunarlander_v2_random"]["terminated"]] == -100).any()
    assert ds["bipedalwalkerhardcore_v3_gait"]["terminated"].any() and ds["bipedalwalker_v3_random"]["terminated"].any()
    assert not ds["bipedalwalker_v3_gait"]["terminated"].any()                    # the gait keeps walking for 500 steps
    assert ds["lunarlander_v2_wind_gravity"]["truncated"].any()                   # TimeLimit 300 reached under wind


def test_box2d_oracles_give_the_same_results_on_any_number_of_threads():
    rng = np.random.default_rng(3)
    for make, act in ((lambda: orc.OracleLunar(37), lambda: rng.integers(0, 4, size=37)),
                      (lambda: orc.OracleLunar(37, continuous=True), lambda: rng.uniform(-1, 1, (37, 2)).astype(np.float32)),
                      (lambda: orc.OracleWalker(37, hardcore=True), lambda: rng.uniform(-1, 1, (37, 4)).astype(np.float32))):
        a, b = make(), make()
        assert np.array_equal(a.reset(seed=8), b.reset(seed=8))
        for t in range(120):
            x = act()
            ra, rb = a.step(x, nthreads=1), b.step(x, nthreads=5)
            assert all(np.array_equal(p, q) for p, q in zip(ra, rb)), t


def test_lunar_reset_draws_are_pinned_to_numpy():
    """LunarLander.reset (lunar_lander.py:325-339,371-377): 12 terrain heights from ONE vectorised uniform(0, H/2,
    size=12), the helipad plateau, the 3-tap smoothing, then the two initial-force draws and the two dispersion draws
    of the embedded step(0) -- the terrain against a numpy Generator, the stream position through the next episode."""
    n = 16
    e = orc.OracleLunar(n)
    e.reset(seed=50)
    H = 400 / 30.0
    for i in range(n):
        g = np.random.Generator(np.random.PCG64(np.random.SeedSequence(50 + i)))
        height = g.uniform(0, H / 2, size=(12,))
        helipad_y = H / 4
        for k in (-2, -1, 0, 1, 2):
            height[11 // 2 + k] = helipad_y
        smooth_y = [0.33 * (height[j - 1] + height[j + 0] + height[j + 1]) for j in range(11)]
        assert np.array_equal(e.terrain(i), np.asarray(smooth_y, dtype=np.float32)), i
    # after the 12 + 2 + 2 draws of reset(), every step draws 2 more: the terrain of the NEXT episode pins the count
    steps = np.zeros(n, dtype=int)
    done_once = np.zeros(n, dtype=bool)
    for t in range(400):
        o, r, te, tr, fo = e.step(np.zeros(n, dtype=np.int64))
        first = (te | tr) & ~done_once
        for i in np.flatnonzero(first):
            g = np.random.Generator(np.random.PCG64(np.random.SeedSequence(50 + i)))
            g.uniform(0, H / 2, size=(12,))
            g.uniform(-1000.0, 1000.0, size=2)          # initial force x, y (two scalar draws)
            g.uniform(-1.0, 1.0, size=2 * (steps[i] + 2))  # dispersion: embedded step(0) + every step so far
            height = g.uniform(0, H / 2, size=(12,))
            for k in (-2, -1, 0, 1, 2):
                height[11 // 2 + k] = H / 4
            smooth_y = [0.33 * (height[j - 1] + height[j + 0] + height[j + 1]) for j in range(11)]
            assert np.array_equal(e.terrain(i), np.asarray(smooth_y, dtype=np.float32)), (i, steps[i])
        done_once |= first
        steps += 1
        if done_once.all():
            break
    assert done_once.all()


@pytest.mark.parametrize("hardcore", [False, True])
def test_walker_rng_stream_position_is_pinned_across_an_episode(hardcore):
    """bipedal_walker.py:404-423,450-452: after the terrain, reset() draws 10 clouds x (1 + 5 x 2) uniforms and one
    hull force; step() draws nothing.  So the terrain of the SECOND episode, generated from the same stream, pins
    every draw in between -- including numpy's half-consumed 32-bit cache left by Generator.integers."""
    n = 12
    e = orc.OracleWalker(n, hardcore=hardcore, max_episode_steps=60)      # the TimeLimit ends the first episode
    e.reset(seed=900)
    for t in range(60):
        o, r, te, tr, fo = e.step(np.zeros((n, 4), dtype=np.float32))
    assert (te | tr).all()
    for i in range(n):
        g = np.random.Generator(np.random.PCG64(np.random.SeedSequence(900 + i)))
        _numpy_terrain(None, hardcore, g)
        for _ in range(200 // 20):
            g.uniform(0, 200)
            for _ in range(5):
                g.uniform(0, 5 * 14 / 30.0)
                g.uniform(0, 5 * 14 / 30.0)
        g.uniform(-5, 5)
        ys, boxes = _numpy_terrain(None, hardcore, g)
        assert np.array_equal(e.terrain(i), ys), i
        assert np.array_equal(e.polys(i), boxes), i


def test_walker_action_arithmetic_follows_numpy_dtype_flow():
    """bipedal_walker.py:528-543,594-596 with a float32 action (the declared action space): motor speed
    `float(SPEED * np.sign(a))`, torque `float(MOTORS_TORQUE * np.clip(np.abs(a), 0, 1))` and -- numpy >= 2 --
    `reward -= 0.00035 * MOTORS_TORQUE * np.clip(np.abs(a), 0, 1)` turning the Python-float reward into a float32
    that the remaining subtractions then stay in."""
    rng = np.random.default_rng(9)
    SPEED = (4, 6, 4, 6)
    for k in range(3000):
        action = rng.uniform(-1.6, 1.6, size=4).astype(np.float32)
        if k % 7 == 0:
            action[rng.integers(0, 4)] = np.float32(0.0)
        delta = float(rng.normal(0, 0.3))
        want_speed = np.array([float(SPEED[j] * np.sign(action[j])) for j in range(4)], dtype=np.float32)
        want_torque = np.array([float(80 * np.clip(np.abs(action[j]), 0, 1)) for j in range(4)], dtype=np.float32)
        reward = delta
        for a in action:
            reward -= 0.00035 * 80 * np.clip(np.abs(a), 0, 1)
        assert isinstance(reward, np.float32)
        ms, mt, r = orc.walker_action_flow(delta, action)
        assert np.array_equal(ms, want_speed) and np.array_equal(mt, want_torque), (k, action)
        assert r == float(reward), (k, action, r, float(reward))
