"""Env snapshots without a GPU: row sizes per kind, header / version / config checks, state_dict round trip and
host-side index validation (gym_b200/snapshot.py, include/b200gym.h: b200gym_snapshot_row_bytes)."""
import pickle

import numpy as np
import pytest

from gym_b200 import _lib, error
from gym_b200.snapshot import FORMAT_VERSION, EnvSnapshot, check_compatible, env_config, host_indices

# PCG64 record 32 B + float64 state + 32-bit Box2D record words + elapsed 4 B + flags 1 B, padded to 32 B
UNPADDED = {
    _lib.KIND_CARTPOLE: 32 + 4 * 8 + 5,
    _lib.KIND_MOUNTAINCAR: 32 + 2 * 8 + 5,
    _lib.KIND_MOUNTAINCAR_CONT: 32 + 2 * 8 + 5,
    _lib.KIND_PENDULUM: 32 + 2 * 8 + 5,
    _lib.KIND_ACROBOT: 32 + 4 * 8 + 5,
    _lib.KIND_LUNARLANDER: 32 + 103 * 4 + 5,
    _lib.KIND_LUNARLANDER_CONT: 32 + 103 * 4 + 5,
    _lib.KIND_BIPEDALWALKER: 32 + 330 * 4 + 5,
    _lib.KIND_BIPEDALWALKER_HARDCORE: 32 + 491 * 4 + 5,
}
ROW_BYTES = {0: 96, 1: 64, 2: 64, 3: 64, 4: 96, 5: 480, 6: 1376, 7: 480, 8: 2016}


@pytest.mark.parametrize("kind", sorted(UNPADDED))
def test_row_bytes_per_kind(kind):
    lib = _lib.load()
    rb = lib.b200gym_snapshot_row_bytes(kind)
    assert rb == ROW_BYTES[kind]
    assert rb % 32 == 0 and rb - 32 < UNPADDED[kind] <= rb


def test_row_bytes_rejects_unknown_kind():
    lib = _lib.load()
    assert lib.b200gym_snapshot_row_bytes(-1) == -1
    assert lib.b200gym_snapshot_row_bytes(9) == -1


def _header(kind=0, row_bytes=96, version=FORMAT_VERSION, **cfg):
    c = env_config(cfg.get("max_episode_steps", 500), cfg.get("autoreset", True), cfg.get("params", [0.0] * 4),
                   cfg.get("flags", 0))
    return {"version": version, "kind": kind, "row_bytes": row_bytes, "config": c}


def test_compatible_header_passes():
    check_compatible(_header(), 0, 96, env_config(500, True, [0.0] * 4, 0))


@pytest.mark.parametrize("bad, match", [
    (dict(version=FORMAT_VERSION + 1), "format version"),
    (dict(version=None), "format version"),
    (dict(kind=4), "kind"),
    (dict(row_bytes=64), "bytes"),
    (dict(max_episode_steps=200), "config"),
    (dict(autoreset=False), "config"),
    (dict(params=[9.8, 0.0, 0.0, 0.0]), "config"),
    (dict(flags=1), "config"),
])
def test_incompatible_header_raises(bad, match):
    with pytest.raises(error.Error, match=match):
        check_compatible(_header(**bad), 0, 96, env_config(500, True, [0.0] * 4, 0))


def test_config_treats_no_limit_as_zero():
    assert env_config(None, 1, (1, 2, 3, 4), 0) == env_config(0, True, [1.0, 2.0, 3.0, 4.0], 0)


def _host_snapshot(m=5, row_bytes=96, d=4):
    rng = np.random.default_rng(0)
    return {"header": _header(row_bytes=row_bytes), "rows": rng.integers(0, 256, (m, row_bytes), dtype=np.uint8),
            "obs": rng.standard_normal((m, d)).astype(np.float32),
            "extras": {"0:RecordEpisodeStatistics": {"ring": np.arange(3, dtype=np.int64), "cur": 1}}}


def test_state_dict_round_trip_through_pickle():
    # from_state_dict moves arrays to a device; with "cpu" the round trip runs without one
    sd = _host_snapshot()
    snap = EnvSnapshot.from_state_dict(pickle.loads(pickle.dumps(sd)), "cpu")
    assert len(snap) == 5 and snap.kind == 0 and snap.version == FORMAT_VERSION
    back = snap.state_dict()
    assert back["header"] == sd["header"]
    np.testing.assert_array_equal(back["rows"], sd["rows"])
    np.testing.assert_array_equal(back["obs"], sd["obs"])
    np.testing.assert_array_equal(back["extras"]["0:RecordEpisodeStatistics"]["ring"], np.arange(3))
    assert back["extras"]["0:RecordEpisodeStatistics"]["cur"] == 1


def test_from_state_dict_rejects_bad_version_and_shapes():
    sd = _host_snapshot()
    sd["header"]["version"] = 0
    with pytest.raises(error.Error, match="format version"):
        EnvSnapshot.from_state_dict(sd, "cpu")
    sd = _host_snapshot()
    sd["rows"] = sd["rows"][:, :64]
    with pytest.raises(error.Error, match="rows"):
        EnvSnapshot.from_state_dict(sd, "cpu")
    sd = _host_snapshot()
    sd["obs"] = sd["obs"][:3]
    with pytest.raises(error.Error, match="observations"):
        EnvSnapshot.from_state_dict(sd, "cpu")


def test_host_indices_validation():
    np.testing.assert_array_equal(host_indices([3, 0, 3], 4, "idx"), np.array([3, 0, 3], dtype=np.int64))
    assert host_indices(np.array([], dtype=np.int64), 4, "idx").dtype == np.int64
    assert host_indices([], 4, "idx").size == 0
    with pytest.raises(error.Error, match="out of range"):
        host_indices([0, 4], 4, "idx")
    with pytest.raises(error.Error, match="out of range"):
        host_indices([-1], 4, "idx")
    with pytest.raises(error.Error, match="integers"):
        host_indices([0.5], 4, "idx")
    with pytest.raises(error.Error, match="1-D"):
        host_indices([[0, 1]], 4, "idx")
