"""The Box2D building blocks on the device (b200gym_selftest_box2d, csrc/b2probe.cu) against float64 geometry and
against the host build of the same source, bit for bit.  `pytest -m gpu`.

The generators and checks are those of tests/test_box2d_geometry_cpu.py (tests/box2d_geometry.py).  On top of them:
b2Distance and b2TimeOfImpact under the contracts of the two oracle tests in test_oracle_box2d.py, and
BipedalWalker's lidar end to end: the 10 fractions of obs[:, 14:24] recomputed in float64 against every terrain edge
and obstacle box, which checks the ray casts and the edge / box windows env_post prunes them to.
"""
import ctypes

import numpy as np
import pytest

import box2d_geometry as g
from hostsim import sim

pytestmark = pytest.mark.gpu


def device_probe(op, records):
    import torch
    from gym_b200 import _lib
    lib = _lib.load()
    rec = torch.as_tensor(np.ascontiguousarray(records, dtype=np.float32).reshape(-1, 16), device="cuda")
    out = torch.empty_like(rec)
    _lib.check(lib.b200gym_selftest_box2d(int(op), ctypes.c_void_p(rec.data_ptr()), rec.shape[0],
                                          ctypes.c_void_p(out.data_ptr()), None))
    torch.cuda.synchronize()
    return out.cpu().numpy()


def probe(op, records):
    """The device's answer, after checking that it equals the host build's bit for bit."""
    dev = device_probe(op, records)
    host = sim.box2d_probe(op, records)
    diff = np.flatnonzero((dev.view(np.uint32) != host.view(np.uint32)).any(axis=1))
    assert diff.size == 0, (op, diff[:5], dev[diff[:2]], host[diff[:2]])
    return dev


@pytest.fixture(scope="module")
def polys():
    return g.fixture_polygons()


def test_rot_of_on_the_device():
    x = g.rot_cases()
    out = probe(g.OP_ROT, g.rot_records(x))
    bad = g.check_rot(x, out)
    assert bad.size == 0, (x[bad[:5]], out[bad[:5], :2])


def test_edge_polygon_manifolds_on_the_device(polys):
    rec, kinds = g.edge_polygon_cases(polys)
    out = probe(g.OP_EDGE_POLYGON, rec)
    bad = g.check_edge_polygon(rec, out, polys)
    assert not bad, (len(bad), bad[:3])
    rng = np.random.default_rng(8)
    keep = (kinds == "parallel") | (kinds == "vertex")
    other = probe(g.OP_EDGE_POLYGON, g.perturbed(rec[keep], rng))
    assert np.array_equal(out[keep][:, [0, 1, 8, 11]].view(np.uint32), other[:, [0, 1, 8, 11]].view(np.uint32))


def test_box_polygon_manifolds_on_the_device(polys):
    rec, _ = g.box_polygon_cases(polys)
    out = probe(g.OP_BOX_POLYGON, rec)
    bad = g.check_box_polygon(rec, out, polys)
    assert not bad, (len(bad), bad[:3])


def test_ray_casts_on_the_device():
    rec = g.edge_ray_cases()
    out = probe(g.OP_EDGE_RAYCAST, rec)
    assert g.check_edge_ray(rec, out).size == 0
    rec = g.box_ray_cases()
    out = probe(g.OP_BOX_RAYCAST, rec)
    assert g.check_box_ray(rec, out).size == 0
    xs, ys, order, p1, p2 = g.nearest_hit_cases()
    frac = g.fold_nearest(probe, xs, ys, order, p1, p2)
    assert np.all(np.abs(frac - g.nearest_hit_reference(xs, ys, p1, p2)) <= 1e-5)


@pytest.mark.parametrize("dim", [2, 3])
def test_solve22_solve33_on_the_device(dim):
    rec, kinds = g.solve_cases()
    out = probe(g.OP_SOLVE22 if dim == 2 else g.OP_SOLVE33, rec)
    assert not g.check_solve(rec, out, dim, kinds)


def test_gjk_distance_on_the_device_matches_brute_force_geometry(polys):
    """test_oracle_box2d.py's b2Distance contract on the device: 3 000 random poses of the lander's hull and leg
    against a segment; the distance is the brute-force polygon-segment distance within 2e-5 (1 + d), 0 when they
    overlap (then GJK ends with a full simplex or within 1e-4)."""
    rng = np.random.default_rng(5)
    recs, want, over = [], [], []
    for k in range(3000):
        f = k % 2
        a = rng.uniform(-3.2, 3.2)
        c = rng.uniform(-2.0, 2.0, 2)
        v1, v2 = rng.uniform(-2.0, 2.0, 2), rng.uniform(-2.0, 2.0, 2)
        if np.linalg.norm(v2 - v1) < 0.2:
            continue
        r = np.zeros(16, dtype=np.float32)
        r[0] = f; r[1:3] = v1; r[3:5] = v2; r[5:7] = c; r[7] = a
        recs.append(r)
    rec = np.stack(recs)
    rot = probe(g.OP_ROT, g.rot_records(rec[:, 7]))
    for i, r in enumerate(rec.astype(np.float64)):
        W = g.transform(polys[int(r[0])], r[5:7], rot[i, :2])
        d = g.polygon_segment_distance(W, r[1:3], r[3:5])
        want.append(d)
        over.append(d == 0.0)
    out = probe(g.OP_GJK, rec)
    got, cnt, want, over = out[:, 0].astype(np.float64), out[:, 1], np.array(want), np.array(over)
    ok_over = (got < 1e-3) & (cnt == 3) | (got < 1e-4)
    ok_sep = (np.abs(got - want) <= 2e-5 + 2e-5 * want) & ((cnt == 1) | (cnt == 2))
    assert np.all(np.where(over, ok_over, ok_sep)), np.flatnonzero(~np.where(over, ok_over, ok_sep))[:5]
    assert over.sum() > 100 and len(rec) > 2500


def test_time_of_impact_on_the_device_lands_on_the_target_separation():
    """test_oracle_box2d.py's b2TimeOfImpact contract on the device: touching at t means the cores are `target`
    +- tolerance apart at the pose interpolated to t (and, without rotation, no sampled earlier time is closer);
    separated means they are further apart than that at the end of the sweep (everywhere, without rotation)."""
    slop = g.LINEAR_SLOP
    target, tol, eps = max(slop, 4 * slop - 3 * slop), 0.25 * slop, 2e-5
    rng = np.random.default_rng(11)
    recs, trans = [], []
    for k in range(4000):
        f = k % 2
        slope = rng.uniform(-0.5, 0.5)
        v1, v2 = (-3.0, -3.0 * slope), (3.0, 3.0 * slope)
        x0 = rng.uniform(-1.0, 1.0)
        c0 = np.array([x0, slope * x0 + rng.uniform(0.7, 1.6)])
        a0 = rng.uniform(-3.0, 3.0)
        c1 = c0 + np.array([rng.normal(0, 0.4), -abs(rng.normal(0, 1.2))])
        spin = rng.normal(0, 0.5)
        translating = k % 4 < 2
        a1 = a0 if translating else a0 + spin
        r = np.zeros(16, dtype=np.float32)
        r[0] = f; r[1:3] = v1; r[3:5] = v2; r[5:7] = c0; r[7] = a0; r[8:10] = c1; r[10] = a1
        recs.append(r)
        trans.append(translating)
    rec, trans = np.stack(recs), np.array(trans)
    out = probe(g.OP_TOI, rec)
    st, t = out[:, 0].astype(int), out[:, 1]

    def dist(betas):
        """GJK distance at the poses interpolated to betas (one per case), as the oracle test computes them."""
        b = np.asarray(betas, dtype=np.float32)[:, None]
        q = np.zeros_like(rec)
        q[:, 0:5] = rec[:, 0:5]
        q[:, 5:7] = ((1 - b) * rec[:, 5:7] + b * rec[:, 8:10]).astype(np.float32)
        q[:, 7] = ((1 - b[:, 0]) * rec[:, 7] + b[:, 0] * rec[:, 10]).astype(np.float32)
        return probe(g.OP_GJK, q)[:, 0]

    assert np.all(np.isin(st, (2, 3, 4))), np.flatnonzero(~np.isin(st, (2, 3, 4)))[:5]
    touch, sep = st == 3, st == 4
    d_t = dist(t)
    start = touch & (t == 0.0)
    assert np.all((d_t[start] > 0) & (d_t[start] <= target + tol + eps))
    mid = touch & (t > 0.0)
    assert np.all(np.abs(d_t[mid] - target) <= tol + eps), np.flatnonzero(mid & (np.abs(d_t - target) > tol + eps))[:5]
    for frac in np.linspace(0.0, 1.0, 12, endpoint=False):
        d = dist(frac * t)
        assert np.all(d[mid & trans] >= target - tol - eps)
    assert np.all(t[sep] == 1.0)
    for b in np.linspace(0.0, 1.0, 16):
        d = dist(np.full(len(rec), b))
        assert np.all(d[sep & (trans | (b == 1.0))] >= target - tol - eps)
    assert (mid.sum() > 800) and (sep.sum() > 800)


@pytest.mark.parametrize("env_id", ["BipedalWalker-v3", "BipedalWalkerHardcore-v3"])
def test_lidar_matches_float64_ray_casts_over_every_terrain_edge_and_box(env_id):
    """obs[:, 14:24] against the float64 nearest hit of each lidar ray over ALL 199 terrain edges (and every obstacle
    box), from the hull's origin xf.p; after random steps, on 384 envs.  The fraction agrees within the float32
    bound of the hit edge (ray_t_bound plus the rounding of coordinates up to 100 m); rays whose nearest hit is
    within that bound of an edge end or of a tie between two edges may pick either side of it."""
    import torch
    import gym_b200
    N = 384
    env = gym_b200.vector.make(env_id, N)
    env.reset(seed=7)
    rng = np.random.default_rng(3)
    lc = sim.shape_verts(2)[1]
    step = np.float32(14 / 30.0)
    xs = np.array([np.float32(k * (14 / 30.0)) for k in range(200)], dtype=np.float64)
    sn = np.sin(1.5 * np.arange(10) / 10.0)
    cs = np.cos(1.5 * np.arange(10) / 10.0)
    checked = 0
    for t in range(60):
        a = rng.uniform(-1, 1, (N, 4)).astype(np.float32)
        obs, *_ = env.step(torch.as_tensor(a, device=env.device))
        if t % 20 != 19:
            continue
        obs = obs.cpu().numpy()
        bodies, _ = env.walker_bodies()
        hull = bodies[:, 0].cpu().numpy()
        terrain, boxes, nbox = (x.cpu().numpy() for x in env.walker_terrain())
        q = probe(g.OP_ROT, g.rot_records(hull[:, 2]))
        qs, qc = q[:, 0], q[:, 1]
        px = hull[:, 0] - (qc * lc[0] - qs * lc[1])          # sync_xf: xf.p = c - rmul(q, localCenter), float32
        py = hull[:, 1] - (qs * lc[0] + qc * lc[1])
        for i in range(N):
            p1 = np.array([px[i], py[i]], dtype=np.float64)
            v1 = np.stack([xs[:-1], terrain[i, :-1]], axis=1).astype(np.float64)
            v2 = np.stack([xs[1:], terrain[i, 1:]], axis=1).astype(np.float64)
            for k in range(10):
                p2 = np.array([np.float32(float(px[i]) + sn[k] * (160 / 30.0)),
                               np.float32(float(py[i]) - cs[k] * (160 / 30.0))], dtype=np.float64)
                P1, P2 = np.broadcast_to(p1, v1.shape), np.broadcast_to(p2, v1.shape)
                tt, ss, den = g.segment_params(v1, v2, P1, P2)
                with np.errstate(invalid="ignore"):
                    tb = g.ray_t_bound(v1 - P1, P2 - P1, tt, den) + 16 * g.U * 100.0 / np.abs(den)
                    hit = (tt >= 0) & (tt <= 1) & (ss >= 0) & (ss <= 1)
                    near = (tt >= -tb) & (tt <= 1 + tb) & (ss >= -1e-5) & (ss <= 1 + 1e-5)
                cand_t = list(tt[hit]) + [1.0]
                lo_t = list(tt[near]) + [1.0]
                tol = float(np.max(tb[near], initial=0.0)) + 1e-7
                for b in range(int(nbox[i])):
                    bx = boxes[i, b].astype(np.float64)[None, :]
                    enter, leave = g.slab(bx, p1[None, :], p2[None, :])
                    if enter[0] > 0 and enter[0] <= leave[0] and enter[0] <= 1:
                        cand_t.append(float(enter[0]))
                    if enter[0] > -1e-5 and enter[0] <= leave[0] + 1e-5 and enter[0] <= 1 + 1e-5:
                        lo_t.append(float(enter[0]))
                        tol = max(tol, 16 * g.U * 100.0 / (160 / 30.0) + 1e-7)
                want_hi, want_lo = min(cand_t), min(lo_t)
                got = float(obs[i, 14 + k])
                assert want_lo - tol <= got <= want_hi + tol, (env_id, t, i, k, got, want_lo, want_hi, tol)
                checked += 1
    assert checked == 3 * N * 10
