"""Kernel B (resident grid, every HBM row moved by bulk copies, results written into the tile's shared-memory stage)
against kernel A (one tile per CTA, plain loads and stores): same per-env arithmetic, so every output and the
persistent state must be bit-identical."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ENV_IDS = ["CartPole-v1", "MountainCar-v0", "MountainCarContinuous-v0", "Pendulum-v1", "Acrobot-v1"]


def _actions(env_id, rng, T, N):
    if env_id.startswith("CartPole"):
        return rng.integers(0, 2, size=(T, N)).astype(np.int64)
    if env_id.startswith(("MountainCar-", "Acrobot")):
        return rng.integers(0, 3, size=(T, N)).astype(np.int64)
    lim = 3.0 if env_id.startswith("Pendulum") else 1.5
    return rng.uniform(-lim, lim, size=(T, N, 1)).astype(np.float32)


# (env_id, tiles per SM): 9 gives each resident CTA at most 3 tiles, so no stage of the ring is ever refilled;
# 49 gives every CTA at least 7 tiles whatever the occupancy (288 threads: at most 7 CTAs per SM), so every one of
# the kBulkStages stages is refilled and its mbarriers complete a second phase
CASES = ([pytest.param(e, 9, id=e) for e in ENV_IDS] +
         [pytest.param(e, 49, id=f"{e}-multi_round") for e in ENV_IDS])


@pytest.mark.parametrize("env_id,tiles_per_sm", CASES)
def test_bulk_kernel_equals_simple_kernel(env_id, tiles_per_sm, monkeypatch):
    """A ragged last tile (kernel A takes it); max_episode_steps=40 makes the whole batch truncate in the same step
    twice -- every warp is dense then and resets inline, through the stage -- and the terminations in between go
    through the deferred list, whose direct stores must land after the tile's bulk stores.  The list never overflows
    here (test_gpu_launch_shapes.py forces that).  The action dtype cycles through int64 / int32 / uint8.  N stays a
    multiple of 16 at 49 tiles per SM: otherwise the float32 action rows of odd steps are not 16-byte aligned and
    kernel P runs instead of B."""
    import torch
    import gym_b200
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    N = 132 * 256 * 9 + 178 if tiles_per_sm == 9 else tiles_per_sm * sms * 256 + 176
    T = 90
    envs = {}
    for k in ("a", "b"):
        monkeypatch.setenv("B200GYM_KERNEL", k)
        envs[k] = gym_b200.vector.make(env_id, N, max_episode_steps=40)
    monkeypatch.delenv("B200GYM_KERNEL")
    ea, eb = envs["a"], envs["b"]
    assert torch.equal(ea.reset(seed=99)[0], eb.reset(seed=99)[0])
    acts = torch.as_tensor(_actions(env_id, np.random.default_rng(11), T, N), device=ea.device)
    dtypes = [torch.int64, torch.int32, torch.uint8] if ea.discrete else [torch.float32]
    n_done = 0
    for t in range(T):
        a = acts[t].to(dtypes[t % len(dtypes)])
        ra, rb = ea.step(a), eb.step(a)
        for x, y in zip(ra[:4], rb[:4]):
            assert torch.equal(x, y), f"kernel b step {t}"
        m = ra[4]["_final_observation"]
        assert torch.equal(m, rb[4]["_final_observation"])
        assert torch.equal(ra[4]["final_observation"][m], rb[4]["final_observation"][m])
        n_done += int(m.sum())
    assert n_done >= 2 * N
    for x, y in zip(ea.get_state(), eb.get_state()):
        assert torch.equal(x, y), "kernel b state"
    for e in envs.values():
        e.close()
