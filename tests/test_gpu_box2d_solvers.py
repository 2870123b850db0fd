"""The Box2D solver steps on the device (b200gym_selftest_box2d, csrc/b2probe.cu): the records of
tests/test_box2d_solvers_cpu.py, bit for bit equal to the host build of the same source, and under the same float64
contracts (tests/box2d_solvers.py).  `pytest -m gpu`.
"""
import numpy as np
import pytest

import box2d_geometry as g
import box2d_solvers as s
from test_gpu_box2d_geometry import probe

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fc():
    return s.fixture_consts(probe)


@pytest.fixture(scope="module")
def jc():
    return s.joint_consts(probe)


@pytest.fixture(scope="module")
def contacts():
    return s.touching_contacts(probe, g.fixture_polygons())


def test_constants_on_the_device(fc, jc):
    assert not s.check_fixture_consts(fc)
    assert not s.check_joint_consts(jc)


def test_contact_steps_on_the_device(contacts, fc):
    init = probe(s.OP_CONTACT_INIT, contacts)
    assert not s.check_contact_init(contacts, init, fc)
    rec = np.concatenate([s.velocity_records(contacts, init), s.block_records(fc)])
    out = probe(s.OP_CONTACT_VELOCITY, rec)
    assert not s.check_contact_velocity(rec, out, fc)
    rec = s.position_records(contacts)
    out = probe(s.OP_CONTACT_POSITION, rec)
    assert not s.check_contact_position(rec, out, fc)
    rec = s.two_point_position_records(contacts)
    out = probe(s.OP_CONTACT_POSITION, rec)
    assert s.check_contact_position_two(rec, out, fc).size == 0


def test_joint_steps_on_the_device(fc, jc):
    rec = s.joint_velocity_records(fc)
    out = probe(s.OP_JOINT_VELOCITY, rec)
    assert not s.check_joint_velocity(rec, out, fc, jc)
    rec = s.joint_position_records(fc, jc)
    out = probe(s.OP_JOINT_POSITION, rec)
    assert not s.check_joint_position(rec, out, fc, jc)


def test_integration_on_the_device(fc):
    rec = s.integrate_records()
    out = probe(s.OP_INTEGRATE, rec)
    assert s.check_integrate(rec, out, fc).size == 0
