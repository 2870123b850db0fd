"""The Box2D solver steps of the device source -- contact masses and world manifold, one contact velocity iteration
(friction, the 1-point solve, the 2-point block LCP and its condition-number fallback), one contact position
iteration, the revolute joint's velocity and position solves, integration with its clamps -- and the host-computed
mass properties, in the host build (tests/hostsim, csrc/b2probe.cuh), against float64 (tests/box2d_solvers.py).

The C oracle and the CUDA source restate Box2D in two copies that are compared bit for bit elsewhere; an error the two
share passes those tests.  These tie each step to its contract instead.  tests/test_gpu_box2d_solvers.py runs the same
records on the device.
"""
import numpy as np
import pytest

import box2d_geometry as g
import box2d_solvers as s
from hostsim import sim

probe = sim.box2d_probe


@pytest.fixture(scope="module")
def fc():
    return s.fixture_consts(probe)


@pytest.fixture(scope="module")
def jc():
    return s.joint_consts(probe)


@pytest.fixture(scope="module")
def contacts():
    return s.touching_contacts(probe, g.fixture_polygons())


def test_mass_properties_match_exact_polygon_integrals(fc):
    """Mass, centroid and inertia of the five fixtures against exact polygon integrals with gym's densities, and their
    friction (box2d_solvers.check_fixture_consts states the bounds)."""
    bad = s.check_fixture_consts(fc)
    assert not bad, bad


def test_joint_constants_are_the_tasks(jc):
    bad = s.check_joint_consts(jc)
    assert not bad, bad


def test_contact_init_matches_float64_world_manifold_and_masses(contacts, fc):
    out = probe(s.OP_CONTACT_INIT, contacts)
    bad = s.check_contact_init(contacts, out, fc)
    assert not bad, (len(bad), bad[:5])
    two = contacts[:, 13] == 2
    # both sides of the condition-number fallback are reached
    assert (out[two, 10] == 2).sum() > 200 and (out[two, 10] == 1).sum() > 20, ((out[two, 10] == 1).sum())
    assert (contacts[:, 4] == 1).sum() > 50 and (contacts[:, 4] == 0).sum() > 500


def test_contact_velocity_iteration_keeps_its_contracts(contacts, fc):
    init = probe(s.OP_CONTACT_INIT, contacts)
    rec = np.concatenate([s.velocity_records(contacts, init), s.block_records(fc)])
    out = probe(s.OP_CONTACT_VELOCITY, rec)
    bad = s.check_contact_velocity(rec, out, fc)
    assert not bad, (len(bad), bad[:5], out[bad[:2]])
    kase = out[:, 7].astype(int)
    for c in (s.ONE_POINT, s.CASE_BOTH, s.CASE_FIRST, s.CASE_SECOND, s.CASE_NEITHER):
        assert (kase == c).sum() > 50, (c, np.bincount(kase + 1))
    # friction clamps on points whose accumulated normal impulses differ
    cone = np.abs(out[:, 5:7]) == (rec[:, 14:15] * rec[:, 10:12])
    assert (cone & (rec[:, 10:11] != rec[:, 11:12]) & (rec[:, 10:12] > 0)).sum() > 100


def test_contact_position_iteration_keeps_its_contracts(contacts, fc):
    rec = s.position_records(contacts)
    out = probe(s.OP_CONTACT_POSITION, rec)
    bad = s.check_contact_position(rec, out, fc)
    assert not bad, (len(bad), bad[:5])
    sep = out[:, 3]
    # the Baumgarte correction is reached unclamped, clamped at 0 and at maxLinearCorrection
    assert ((sep > -1.0) & (sep < -s.LINEAR_SLOP)).sum() > 500 and (sep > 0).sum() > 100 and (sep < -1.1).sum() > 100


def test_two_point_contact_position_iteration_solves_each_point_at_the_pose_the_first_leaves(contacts, fc):
    rec = s.two_point_position_records(contacts)
    out = probe(s.OP_CONTACT_POSITION, rec)
    bad = s.check_contact_position_two(rec, out, fc)
    assert bad.size == 0, (len(bad), bad[:5], rec[bad[:2]], out[bad[:2]])
    # the first point's correction moves the body, and the second point's separation is the smaller in some records
    _, _, sep, imps = s.position_chain_reference(rec, fc)
    assert (imps[0] > 1e-3).sum() > 100 and (imps[1] > 1e-3).sum() > 100
    r = rec.copy()
    r[:, 13] = 1
    first = probe(s.OP_CONTACT_POSITION, r)[:, 3]
    assert (out[:, 3] < first).sum() > 50


def test_joint_velocity_solve_keeps_its_contracts(fc, jc):
    rec = s.joint_velocity_records(fc)
    out = probe(s.OP_JOINT_VELOCITY, rec)
    bad = s.check_joint_velocity(rec, out, fc, jc)
    assert not bad, (len(bad), bad[:5], rec[bad[:2]], out[bad[:2]])
    st = out[:, 10]
    at_limit = rec[:, 4] == 0
    for j in range(6):
        mine = rec[:, 0] == j
        assert all((mine & (st == k)).sum() > 50 for k in (0, 1, 2)), j
        # exactly at each limit: the limit is active
        lo, hi = np.float32(s.JOINT_DEFS[j][2]), np.float32(s.JOINT_DEFS[j][3])
        assert (mine & at_limit & (rec[:, 8] == lo)).sum() > 20 and (mine & at_limit & (rec[:, 8] == hi)).sum() > 20
    # the warm start keeps a limit impulse, and drops one on a change of limit state
    prev = rec[:, 15]
    assert ((st != 0) & (st == prev) & (out[:, 13] != 0)).sum() > 500
    assert ((st != 0) & (st != prev) & (rec[:, 11] != 0)).sum() > 500
    # the reduced re-solve (a limit impulse brought to 0 at an active limit) and a saturated motor are both reached
    assert ((st != 0) & (out[:, 8] == 0)).sum() > 100
    assert (np.abs(out[:, 9]) == (np.float32(s.DT) * rec[:, 14])).sum() > 1000


def test_joint_position_solve_keeps_its_contracts(fc, jc):
    rec = s.joint_position_records(fc, jc)
    out = probe(s.OP_JOINT_POSITION, rec)
    bad = s.check_joint_position(rec, out, fc, jc)
    assert not bad, (len(bad), bad[:5], rec[bad[:2]], out[bad[:2]])
    assert (out[:, 6] == 1).sum() > 100 and (out[:, 6] == 0).sum() > 1000


def test_integration_matches_float64_with_both_clamps(fc):
    rec = s.integrate_records()
    out = probe(s.OP_INTEGRATE, rec)
    bad = s.check_integrate(rec, out, fc)
    assert bad.size == 0, (bad[:5], rec[bad[:2]], out[bad[:2]])
