"""Sharding a global batch of environments over the GPUs of one node.

The reference has no distributed code: its only "gather" is AsyncVectorEnv
collecting per-worker results over pipes / shared memory
(gym/vector/async_vector_env.py:319-328, gym/vector/utils/shared_memory.py:164-170).
The H100-native equivalent (SURVEY.md 8e): one process per GPU, rank r owns the
contiguous global envs [r*n, (r+1)*n); env i is seeded ``seed + i`` with its
GLOBAL index, so results do not depend on the number of GPUs; every step the
ranks exchange (obs, reward, terminated, truncated) with ONE in-place
all-gather per tensor over NVLink (``torch.distributed``, NCCL backend).

The step kernel writes straight into this rank's slice of the gather buffers
(the "pack" is fused into the kernel's stores), so the all-gather is in place
and there is no extra copy pass.
"""
import torch
import torch.distributed as dist


def shard_range(total, world_size, rank):
    """Contiguous block partition of `total` envs: (first_index, count) of `rank`."""
    if total % world_size != 0:
        raise ValueError(f"num_envs={total} must be divisible by world_size={world_size}")
    n = total // world_size
    return rank * n, n


class GatherBuffers:
    """Global (world*n, ...) result tensors plus this rank's writable slices.

    Works on any device/backend (NCCL on GPUs, gloo on CPU in the tests).
    """

    FIELDS = (("obs", torch.float32), ("reward", torch.float64),
              ("terminated", torch.bool), ("truncated", torch.bool))

    def __init__(self, world_size, rank, n_local, obs_dim, device):
        self.world_size, self.rank, self.n_local = world_size, rank, n_local
        total = world_size * n_local
        self.glob = {
            "obs": torch.zeros((total, obs_dim), dtype=torch.float32, device=device),
            "reward": torch.zeros((total,), dtype=torch.float64, device=device),
            "terminated": torch.zeros((total,), dtype=torch.bool, device=device),
            "truncated": torch.zeros((total,), dtype=torch.bool, device=device),
        }
        lo, hi = rank * n_local, (rank + 1) * n_local
        self.local = {k: v[lo:hi] for k, v in self.glob.items()}

    def all_gather(self, group=None):
        """In-place all-gather of the four result tensors (input = this rank's slice)."""
        if self.world_size == 1:
            return self.glob
        for name, _ in self.FIELDS:
            out, inp = self.glob[name], self.local[name]
            if out.dtype == torch.bool:  # collectives want a numeric dtype; same bytes
                out, inp = out.view(torch.uint8), inp.view(torch.uint8)
            dist.all_gather_into_tensor(out, inp, group=group)
        return self.glob


class _DeviceMemory:
    """Raw device memory exposed through __cuda_array_interface__ (zero-copy torch view)."""

    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (int(ptr), False),
                                         "version": 2, "strides": None}


class P2PGather:
    """The fused step + all-gather path (``b200gym_step_p2p``): peers' gather buffers are mapped
    through CUDA IPC and the step kernel stores every result into all of them over NVLink."""

    def __init__(self, env, world_size, rank, group=None):
        import ctypes

        from gym_b200 import _lib
        self.env = env
        lib = env._lib
        handle = (ctypes.c_ubyte * 64)()
        layout = _lib.P2PLayout()
        with torch.cuda.device(env.device):
            _lib.check(lib.b200gym_p2p_create(env._handle, world_size, rank, ctypes.cast(handle, ctypes.c_void_p),
                                              ctypes.cast(ctypes.pointer(layout), ctypes.c_void_p)), env._handle)
            mine = torch.tensor(list(bytes(handle)), dtype=torch.uint8, device=env.device)
            allh = torch.empty(world_size * 64, dtype=torch.uint8, device=env.device)
            if world_size > 1:
                dist.all_gather_into_tensor(allh, mine, group=group)
            else:
                allh.copy_(mine)
            blob = ctypes.create_string_buffer(allh.cpu().numpy().tobytes(), world_size * 64)
            _lib.check(lib.b200gym_p2p_connect(env._handle, ctypes.cast(blob, ctypes.c_void_p)), env._handle)
        rows, d = int(layout.rows), env.obs_dim
        self.sets = []
        for s in range(2):
            b = layout.base + s * layout.set_bytes

            def view(off, shape, typestr, dtype=None):
                t = torch.as_tensor(_DeviceMemory(b + off, shape, typestr), device=env.device)
                return t if dtype is None else t.view(dtype)

            self.sets.append({
                "obs": view(layout.off_obs, (rows, d), "<f4"),
                "reward": view(layout.off_reward, (rows,), "<f8"),
                "terminated": view(layout.off_terminated, (rows,), "|u1", torch.bool),
                "truncated": view(layout.off_truncated, (rows,), "|u1", torch.bool),
            })
        self.final_obs = [torch.zeros((env.num_envs, d), dtype=torch.float32, device=env.device) for _ in range(2)]

    def step(self, actions):
        import ctypes

        from gym_b200 import _lib
        env = self.env
        act, code = env._device_actions(actions)
        which = ctypes.c_int(0)
        fo = self.final_obs[0]
        self.final_obs.reverse()
        _lib.check(env._lib.b200gym_step_p2p(env._handle, ctypes.c_void_p(act.data_ptr()), code,
                                             ctypes.c_void_p(fo.data_ptr()), env._stream(), ctypes.byref(which)),
                   env._handle)
        self._keep = act
        return self.sets[which.value], fo


class ShardedVectorEnv:
    """This rank's shard of a global ``B200VectorEnv`` batch + per-step all-gather.

    ``step(actions_local)`` takes the actions of this rank's envs (a replicated
    policy only needs its own slice) and returns the GLOBAL
    (obs, rewards, terminateds, truncateds) tensors, identical on every rank.

    gather: "p2p"  -- fused: the step kernel stores into every peer's buffers over NVLink
                      (CUDA IPC peer memory) and a flag exchange ends the step;
            "nccl" -- the step kernel writes this rank's slice, then one in-place NCCL
                      all-gather per result tensor (the baseline the fused path is measured against);
            None   -- no exchange (each rank only sees its own slice filled in).
    """

    def __init__(self, env_id, total_envs, group=None, gather="nccl", **kwargs):
        from gym_b200.vector_env import B200VectorEnv
        if gather is True:
            gather = "nccl"
        if gather not in ("p2p", "nccl", None, False):
            raise ValueError("gather must be 'p2p', 'nccl' or None")
        if kwargs.get("wrappers"):
            raise ValueError("ShardedVectorEnv does not take per-env wrappers")
        self.group = group
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.world_size = dist.get_world_size(group) if dist.is_initialized() else 1
        self.first_index, self.n_local = shard_range(total_envs, self.world_size, self.rank)
        self.total_envs = total_envs
        self.gather = gather or None
        self.env = B200VectorEnv(env_id, self.n_local, first_index=self.first_index, **kwargs)
        # two sets of gather buffers, alternating like the env's own double buffering
        self.buffers = [GatherBuffers(self.world_size, self.rank, self.n_local, self.env.obs_dim, self.env.device)
                        for _ in range(2)]
        for k in range(2):
            self.env._out[k].update(self.buffers[k].local)  # kernel writes into the gather slices
        self.p2p = P2PGather(self.env, self.world_size, self.rank, group) if self.gather == "p2p" else None
        self.num_envs = total_envs
        self.single_observation_space = self.env.single_observation_space
        self.single_action_space = self.env.single_action_space

    def _finish(self):
        buf = self.buffers[self.env._flip]
        return buf.all_gather(self.group) if self.gather else buf.glob

    def _no_capture(self, what):
        from gym_b200.vector_env import refuse_capture
        refuse_capture(f"ShardedVectorEnv.{what}()", "multi-GPU capture is not supported")

    def reset(self, *, seed=None, options=None):
        self._no_capture("reset")
        # reset is off the hot path: always exchanged with the plain all-gather
        self.env.reset(seed=seed, options=options)
        return self._finish()["obs"], {}

    def step(self, actions_local):
        self._no_capture("step")
        if self.p2p is not None:
            from gym_b200 import error
            from gym_b200.vector_env import FinalInfos
            self.env._assert_open("step")
            if not self.env._has_reset:
                raise error.ResetNeeded("Cannot call env.step() before calling env.reset()")
            g, final_obs = self.p2p.step(actions_local)
            lo, hi = self.first_index, self.first_index + self.n_local
            infos = FinalInfos(final_obs, g["terminated"][lo:hi], g["truncated"][lo:hi])
            return g["obs"], g["reward"], g["terminated"], g["truncated"], infos
        _, _, _, _, infos = self.env.step(actions_local)
        g = self._finish()
        return g["obs"], g["reward"], g["terminated"], g["truncated"], infos

    def _no_snapshots(self, what):
        from gym_b200 import error
        raise error.Error(f"ShardedVectorEnv does not support {what}(): its gathered global results would be stale "
                          "after a restore or clone")

    def snapshot(self, indices=None):
        self._no_snapshots("snapshot")

    def restore(self, snap, indices=None):
        self._no_snapshots("restore")

    def clone(self, src):
        self._no_snapshots("clone")

    def close(self):
        self.env.close()
