"""``EnvSnapshot`` -- the per-env state of a ``B200VectorEnv`` taken out of the engine and put back.

A snapshot holds, for each env it covers, one device row of ``b200gym_snapshot_row_bytes(kind)`` bytes with
everything the engine owns for that env (include/b200gym.h: PCG64 stream, state, TimeLimit counter, plain-Env flag,
and for the Box2D kinds the whole solver record), the observation last returned for it, and a header naming the
format version, the kind and the construction config.  Rows only mean something to an env of the same kind and
config; ``check_compatible`` refuses anything else.  ``state_dict()`` / ``from_state_dict()`` move a snapshot through
host memory (numpy arrays), which is what pickling an env uses.
"""
import numpy as np

from gym_b200 import error

FORMAT_VERSION = 1


def _torch():
    import torch
    return torch


def env_config(max_episode_steps, autoreset, params, flags):
    """The construction config a snapshot is tied to, in a form that compares and pickles."""
    return {"max_episode_steps": int(max_episode_steps or 0), "autoreset": bool(autoreset),
            "params": [float(p) for p in params], "flags": int(flags)}


def check_compatible(header, kind, row_bytes, config):
    """Raise ``error.Error`` unless a snapshot with ``header`` can be loaded into an env of this kind and config."""
    if header.get("version") != FORMAT_VERSION:
        raise error.Error(f"snapshot format version {header.get('version')!r} is not supported "
                          f"(this build reads version {FORMAT_VERSION})")
    if header.get("kind") != kind:
        raise error.Error(f"snapshot of env kind {header.get('kind')} cannot be loaded into an env of kind {kind}")
    if header.get("row_bytes") != row_bytes:
        raise error.Error(f"snapshot rows of {header.get('row_bytes')} bytes do not match this build's "
                          f"{row_bytes}-byte rows")
    if header.get("config") != config:
        raise error.Error(f"snapshot was taken with config {header.get('config')}, this env has {config}")


def host_indices(indices, n, what):
    """Host-side index validation: a list / numpy array of env indices -> int64 numpy array, every entry in [0, n)."""
    idx = np.asarray(indices)
    if idx.ndim != 1 or not (np.issubdtype(idx.dtype, np.integer) or idx.size == 0):
        raise error.Error(f"{what} must be a 1-D sequence of integers, got shape {idx.shape} and dtype {idx.dtype}")
    idx = idx.astype(np.int64, copy=False)
    if idx.size and (idx.min() < 0 or idx.max() >= n):
        bad = idx[(idx < 0) | (idx >= n)][0]
        raise error.Error(f"{what}: index {int(bad)} is out of range for {n} envs")
    return np.ascontiguousarray(idx)


class EnvSnapshot:
    """Device rows + last observations + header of some envs of a ``B200VectorEnv`` (see the module docstring).

    ``extras`` carries the per-snapshot state of wrappers (``gym_b200.wrappers``), keyed by wrapper layer."""

    def __init__(self, header, rows, obs, extras=None):
        self.header = dict(header)
        self.rows = rows          # torch uint8 (m, row_bytes), 128-byte aligned
        self.obs = obs            # torch float32 (m, obs_dim)
        self.extras = {} if extras is None else extras

    def __len__(self):
        return int(self.rows.shape[0])

    @property
    def kind(self):
        return self.header["kind"]

    @property
    def version(self):
        return self.header["version"]

    def state_dict(self):
        """Host copy: {"header": dict, "rows": uint8 (m, row_bytes), "obs": float32 (m, D), "extras": {...}}."""
        torch = _torch()

        def host(v):
            return v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else v

        return {"header": dict(self.header), "rows": host(self.rows), "obs": host(self.obs),
                "extras": {k: {kk: host(vv) for kk, vv in e.items()} for k, e in self.extras.items()}}

    @classmethod
    def from_state_dict(cls, state, device):
        """Inverse of ``state_dict``; the arrays go to CUDA device ``device``."""
        torch = _torch()
        header = dict(state["header"])
        if header.get("version") != FORMAT_VERSION:
            raise error.Error(f"snapshot format version {header.get('version')!r} is not supported "
                              f"(this build reads version {FORMAT_VERSION})")
        rows = np.ascontiguousarray(state["rows"], dtype=np.uint8)
        if rows.ndim != 2 or rows.shape[1] != header.get("row_bytes"):
            raise error.Error(f"snapshot rows of shape {rows.shape} do not match the header's "
                              f"{header.get('row_bytes')}-byte rows")

        def dev(v):
            return torch.from_numpy(np.ascontiguousarray(v)).to(device) if isinstance(v, np.ndarray) else v

        obs = np.ascontiguousarray(state["obs"], dtype=np.float32)
        if obs.shape[0] != rows.shape[0]:
            raise error.Error(f"snapshot holds {rows.shape[0]} rows but {obs.shape[0]} observations")
        extras = {k: {kk: dev(vv) for kk, vv in e.items()} for k, e in state.get("extras", {}).items()}
        return cls(header, dev(rows), dev(obs), extras)
