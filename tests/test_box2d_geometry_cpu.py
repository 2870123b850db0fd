"""The Box2D building blocks of the device source -- rot_of, the edge-polygon and box-polygon manifolds, the edge and
box ray casts, b2Distance, b2TimeOfImpact, solve22 / solve33 -- in the host build (tests/hostsim, csrc/b2probe.cuh),
against float64 geometry (tests/box2d_geometry.py).

The C oracle and the CUDA source restate Box2D in two copies that are compared bit for bit elsewhere; an error the two
share passes those tests.  These tie each block to plain geometry instead, at the inputs where geometry code goes
wrong: parallel faces, vertices on edges, rays through edge ends or parallel to them, zero denominators, quadrant
switches.  tests/test_gpu_box2d_geometry.py runs the same generators on the device.
"""
import numpy as np
import pytest

import box2d_geometry as g
from hostsim import sim

probe = sim.box2d_probe


@pytest.fixture(scope="module")
def polys():
    return g.fixture_polygons()


def test_rot_of_is_within_its_derived_bound_of_float64_sin_cos():
    x = g.rot_cases()
    out = probe(g.OP_ROT, g.rot_records(x))
    bad = g.check_rot(x, out)
    assert bad.size == 0, (x[bad[:5]], out[bad[:5], :2])
    # the signed zeros come back as sin 0 = 0, cos 0 = 1 (the sign of rot_of(-0).s is not kept: +0)
    z = probe(g.OP_ROT, g.rot_records(np.array([0.0, -0.0], dtype=np.float32)))
    assert (z[:, 0] == 0.0).all() and (z[:, 1] == 1.0).all()


def test_edge_polygon_manifolds_agree_with_float64_geometry(polys):
    rec, kinds = g.edge_polygon_cases(polys)
    out = probe(g.OP_EDGE_POLYGON, rec)
    bad = g.check_edge_polygon(rec, out, polys)
    assert not bad, (len(bad), bad[:3], kinds[[b[0] for b in bad[:3]]])
    counts = out[:, 1]
    # the constructed families do what they were built for
    assert (counts[kinds == "parallel"] == 2).mean() > 0.7
    assert (counts[kinds == "vertex"] >= 1).all()
    assert (counts[kinds == "past_end"] == 0).all()
    assert (out[:, 0][counts > 0] == 1).sum() > 50 and (out[:, 0][counts > 0] == 0).sum() > 500


def test_edge_polygon_feature_ids_are_stable_under_one_ulp_pose_changes(polys):
    rec, kinds = g.edge_polygon_cases(polys)
    keep = (kinds == "parallel") | (kinds == "vertex")
    rec = rec[keep]
    base = probe(g.OP_EDGE_POLYGON, rec)
    rng = np.random.default_rng(8)
    for _ in range(3):
        other = probe(g.OP_EDGE_POLYGON, g.perturbed(rec, rng))
        same = (base[:, 0:2] == other[:, 0:2]).all(axis=1)
        ids = base[:, 8:12:3].view(np.uint32) == other[:, 8:12:3].view(np.uint32)
        ok = same & (ids[:, 0] | (base[:, 1] < 1)) & (ids[:, 1] | (base[:, 1] < 2))
        assert ok.all(), np.flatnonzero(~ok)[:5]


def test_box_polygon_manifolds_agree_with_float64_geometry(polys):
    rec, kinds = g.box_polygon_cases(polys)
    out = probe(g.OP_BOX_POLYGON, rec)
    bad = g.check_box_polygon(rec, out, polys)
    assert not bad, (len(bad), bad[:3])
    assert (out[:, 1] > 0).sum() > 500 and (out[:, 1] == 2).sum() > 100


def test_edge_ray_cast_agrees_with_float64_segment_intersection():
    rec = g.edge_ray_cases()
    out = probe(g.OP_EDGE_RAYCAST, rec)
    bad = g.check_edge_ray(rec, out)
    assert bad.size == 0, (bad[:5], rec[bad[:5]], out[bad[:5], :2])
    assert (out[:, 0] == 1).sum() > 2000
    # a ray starting on the edge hits at t = 0; a ray parallel to it never hits
    on = probe(g.OP_EDGE_RAYCAST, np.array([[-1, 0.5, 1, 0.5, 0, 0.5, 0.3, -1, 1] + [0] * 7], dtype=np.float32))
    par = probe(g.OP_EDGE_RAYCAST, np.array([[-1, 0.5, 1, 0.5, -2, 0.5, 2, 0.5, 1] + [0] * 7], dtype=np.float32))
    assert on[0, 0] == 1 and on[0, 1] == 0.0 and par[0, 0] == 0


def test_box_ray_cast_agrees_with_float64_slab_intersection():
    rec = g.box_ray_cases()
    out = probe(g.OP_BOX_RAYCAST, rec)
    bad = g.check_box_ray(rec, out)
    assert bad.size == 0, (bad[:5], rec[bad[:5]], out[bad[:5], :2])
    assert (out[:, 0] == 1).sum() > 2000


def test_ray_cast_with_max_fraction_clipping_keeps_the_nearest_hit():
    xs, ys, order, p1, p2 = g.nearest_hit_cases()
    frac = g.fold_nearest(probe, xs, ys, order, p1, p2)
    want = g.nearest_hit_reference(xs, ys, p1, p2)
    assert np.all(np.abs(frac - want) <= 1e-5), np.flatnonzero(np.abs(frac - want) > 1e-5)[:5]


@pytest.mark.parametrize("dim", [2, 3])
def test_solve22_solve33_are_within_the_forward_error_bound(dim):
    rec, kinds = g.solve_cases()
    out = probe(g.OP_SOLVE22 if dim == 2 else g.OP_SOLVE33, rec)
    bad = g.check_solve(rec, out, dim, kinds)
    assert not bad, (len(bad), bad[:5], kinds[bad[:5]])
