"""The Box2D step (step kernel -> TOI kernel over the parked envs -> compacted reset-list kernel, DESIGN.md §4.4) at
the launch shapes bench.py times, 2^16 envs after random play, where its TOI and reset passes take branches that
batches of 1 024 envs never reach:
- TOI warps with several lanes.  The TOI grid is min(count, 12 x SMs) one-warp CTAs, and each warp takes
  L = clamp(ceil(parked / grid), 1, 32) parked envs: L >= 2 (the warp-synchronous rounds of b2l::solve_toi combine
  envs) once more envs are parked than there are warps, and above 32 x grid parked envs the warps go round again.
- The reset-list kernels run at most 2 x SMs CTAs of 128 threads; a step with more resets than threads gives a thread
  a second entry.
- The host path (numpy backend) splits the batch into chunks on two streams.  Each chunk has its own counter slot,
  starts its lists at a non-zero first env, and shares the side buffer of the parked envs with the chunk that runs
  beside it.

Every case runs the default configuration, the three other B200GYM_BOX2D_TOI_DEFER x B200GYM_BOX2D_DEFER settings and
the host path in lockstep, bit for bit on every row of every step and in a snapshot of every env at the end, and
three windows of the batch (the first, the middle and the last envs) against the CPU oracle.  Each case asserts the
branch it claims through b200gym_box2d_list_counts.
"""
import concurrent.futures
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

NTHREADS = os.cpu_count() or 1
KNOBS = ("B200GYM_BOX2D_TOI_DEFER", "B200GYM_BOX2D_DEFER", "B200GYM_HOST_CHUNKS")
TOI_CTAS_PER_SM = 12                  # kToiCtasPerSm (gym_b200/csrc/b200gym.cu): one-warp CTAs of the TOI kernels
RESET_CTAS_PER_SM, RESET_THREADS = 2, 128   # grid cap and CTA size of the reset-list kernels
HOST_TILE = 256                       # the host path's chunks are whole multiples of this many envs
LUNAR_W_BODY = 0                      # lunar::W_BODY: 3 bodies x {c.x, c.y, a, v.x, v.y, w, sleepTime}
WARMUP = 250                          # bench.py's warm-up of the Box2D tasks

# The device configurations; the first is the default and the reference of the others.
DEVICE_CONFIGS = [
    ("default", {}),
    ("toi_inline", {"B200GYM_BOX2D_TOI_DEFER": "0"}),
    ("reset_inline", {"B200GYM_BOX2D_DEFER": "0"}),      # the only path where an autoreset runs inside a TOI warp
    ("all_inline", {"B200GYM_BOX2D_TOI_DEFER": "0", "B200GYM_BOX2D_DEFER": "0"}),
]


def _torch():
    import torch
    return torch


def _sms():
    return _torch().cuda.get_device_properties(0).multi_processor_count


def _lanes(parked, grid):
    """toi_lanes_per_warp: parked envs per TOI warp"""
    return max(1, min(32, -(-parked // grid)))


class _Engine:
    """One engine configuration.  Its knobs are set while it is built and while it is called: the defer knobs are
    read at construction, B200GYM_HOST_CHUNKS at every host step."""

    def __init__(self, name, env_id, n, knobs, host=False, **kwargs):
        import gym_b200
        self.name, self.knobs, self.host = name, dict(knobs), host
        if host:
            kwargs.update(backend="numpy", copy=False, dense_infos=True)
        self.env = self.call(gym_b200.vector.make, env_id, n, **kwargs)
        self.toi_deferred = self.knobs.get("B200GYM_BOX2D_TOI_DEFER", "1") == "1"
        self.reset_deferred = self.knobs.get("B200GYM_BOX2D_DEFER", "1") == "1"

    def call(self, fn, *args, **kwargs):
        with pytest.MonkeyPatch.context() as mp:
            for k in KNOBS:
                mp.delenv(k, raising=False)
            for k, v in self.knobs.items():
                mp.setenv(k, v)
            return fn(*args, **kwargs)

    def slots(self):
        """launch ranges of one step: the chunks of the host path, split as b200gym_step_host splits them"""
        if not self.host:
            return 1
        n, c = self.env.num_envs, int(self.knobs["B200GYM_HOST_CHUNKS"])
        per = -(-(-(-n // c)) // HOST_TILE) * HOST_TILE
        return -(-n // per)

    def step(self, a_dev, a_host):
        """-> (obs, reward, terminated, truncated, final_observation mask, final_observation) as device tensors"""
        torch = _torch()
        o, r, te, tr, info = self.call(self.env.step, a_host if self.host else a_dev)
        out = (o, r, te, tr, info["_final_observation"], info["final_observation"])
        if self.host:
            out = tuple(torch.from_numpy(np.asarray(x)).to(a_dev.device) for x in out)
        return out

    def counts(self):
        return self.env.box2d_list_counts(self.slots())


def _bits(x):
    torch = _torch()
    if x.dtype == torch.float32:
        return x.view(torch.int32)
    if x.dtype == torch.float64:
        return x.view(torch.int64)
    return x


def _differ(x, y):
    torch = _torch()
    d = _bits(x) != _bits(y)
    if d.dim() > 1:
        d = d.flatten(1).any(dim=1)
    rows = torch.nonzero(d).flatten()
    return f"{rows.numel()} rows differ, first {rows[:4].tolist()}"


def _snapshot_words_differ(a, b):
    """{32-bit word of the snapshot row: number of envs in which it differs} of two snapshots of the same batch"""
    torch = _torch()
    d = a.rows.view(torch.int32) != b.rows.view(torch.int32)
    return {int(w): int(d[:, w].sum()) for w in torch.nonzero(d.any(dim=0)).flatten()}


def _assert_same(ref, got, what):
    """One step of two engines, every output bit for bit, the final_observation rows under the mask included."""
    torch = _torch()
    for name, x, y in zip(("obs", "reward", "terminated", "truncated", "final_observation mask"), ref[:5], got[:5]):
        assert torch.equal(_bits(x), _bits(y)), f"{what}: {name}: {_differ(x, y)}"
    m = ref[4]
    assert torch.equal(_bits(ref[5][m]), _bits(got[5][m])), f"{what}: final_observation rows"


class _Windows:
    """Three oracles of m envs standing in for envs [lo, lo + m) of the batch: the first, the middle and the last
    m envs (the last window holds the ragged tail of the step kernel's grid and of the last host chunk)."""

    def __init__(self, make_oracle, n, m):
        self.m = m
        self.los = [0, (n - m) // 2, n - m]
        self.orcs = [make_oracle(m) for _ in self.los]

    def reset(self, seed):
        return [orc.reset(seed=seed, first=lo) for lo, orc in zip(self.los, self.orcs)]

    def step(self, a_host):
        return [orc.step(a_host[lo:lo + self.m], nthreads=NTHREADS) for lo, orc in zip(self.los, self.orcs)]

    def check(self, out, refs, what):
        """The default engine's step (host arrays) against the oracles', bit for bit as test_gpu_lunar.py does."""
        o, r, te, tr, mask, fo = out
        for lo, ref in zip(self.los, refs):
            sl = slice(lo, lo + self.m)
            ro, rr, rte, rtr, rfo = ref
            w = f"{what}, window {lo}"
            assert np.array_equal(te[sl], rte), f"{w}: {np.count_nonzero(te[sl] != rte)} terminated differ"
            assert np.array_equal(tr[sl], rtr), f"{w}: {np.count_nonzero(tr[sl] != rtr)} truncated differ"
            if not np.array_equal(o[sl], ro):
                bad = np.argwhere(o[sl] != ro)
                raise AssertionError(f"{w}: {len(bad)} observation values differ, first env {lo + bad[0][0]}")
            assert np.array_equal(r[sl], rr), f"{w}: reward"
            done = rte | rtr
            assert np.array_equal(mask[sl], done), f"{w}: final_observation mask"
            assert np.array_equal(fo[sl][done], rfo[done]), f"{w}: final_observation rows"

    def close(self):
        for orc in self.orcs:
            orc.close()


def _random_actions(env_id, n, rng):
    if env_id.startswith("LunarLanderContinuous"):
        return rng.uniform(-1.0, 1.0, size=(n, 2)).astype(np.float32)
    if env_id.startswith("LunarLander"):
        return rng.integers(0, 4, size=n).astype(np.int64)
    return rng.uniform(-1.0, 1.0, size=(n, 4)).astype(np.float32)


def _make_oracle(env_id, max_episode_steps):
    from oracle.oracle import OracleLunar, OracleWalker
    if env_id.startswith("LunarLander"):
        return lambda m: OracleLunar(m, max_episode_steps=max_episode_steps, continuous="Continuous" in env_id)
    return lambda m: OracleWalker(m, max_episode_steps=max_episode_steps, hardcore="Hardcore" in env_id)


def _force_falls(engines, windows, mask, vy):
    """Envs `mask` of every engine and of the oracle windows: v = (0, vy) and w = 0 on all three bodies."""
    torch = _torch()
    env = engines[0].env
    snap = env.snapshot()
    words = snap.rows.view(torch.float32)
    rec = 8 + 2 * env._lib.b200gym_state_dim(env.kind)   # the record follows the PCG64 words and the float64 state
    idx = torch.as_tensor(np.flatnonzero(mask), device=env.device)
    for b in range(3):
        w = rec + LUNAR_W_BODY + 7 * b
        words[idx, w + 3] = 0.0
        words[idx, w + 4] = vy
        words[idx, w + 5] = 0.0
    for e in engines:
        e.call(e.env.restore, snap)
    for lo, orc in zip(windows.los, windows.orcs):
        for k in np.flatnonzero(mask[lo:lo + windows.m]):
            for b in range(3):
                orc.set_body_velocity(int(k), b, 0.0, vy, 0.0)
    bodies, flags = env.lunar_bodies()
    bodies, flags = bodies.cpu().numpy(), flags.cpu().numpy()
    for lo, orc in zip(windows.los, windows.orcs):
        for k in range(windows.m):
            ob, of = orc.bodies(k)
            assert np.array_equal(bodies[lo + k], ob), f"env {lo + k}: bodies after the edit"
            assert flags[lo + k, :3].tolist() == of[:3].tolist() and flags[lo + k, 5] == of[5], f"env {lo + k}"


def _run(case, env_id, n, steps, m, host64=False, max_episode_steps=None, force=None, seed=0):
    """All engine configurations in lockstep from reset(seed) under random actions (a pool of 8 batches drawn on the
    host, cycled as bench.py cycles its pool) or, with `force` = (mask, vy), action 0 after the falls of `mask` were
    forced.  Returns the list counts: per step (parked, resets) of the device path, and per host configuration the
    largest count of each chunk."""
    torch = _torch()
    dev = torch.device("cuda", 0)
    kw = {} if max_episode_steps is None else dict(max_episode_steps=max_episode_steps)
    engines = [_Engine(name, env_id, n, knobs, **kw) for name, knobs in DEVICE_CONFIGS]
    engines.append(_Engine("host_5", env_id, n, {"B200GYM_HOST_CHUNKS": "5"}, host=True, **kw))
    if host64:
        engines.append(_Engine("host_64", env_id, n, {"B200GYM_HOST_CHUNKS": "64"}, host=True, **kw))
    windows = _Windows(_make_oracle(env_id, engines[0].env.max_episode_steps), n, m)
    steps_counts = []
    chunk_max = {e.name: (np.zeros(e.slots(), np.int64), np.zeros(e.slots(), np.int64)) for e in engines if e.host}
    try:
        obs0 = [e.call(e.env.reset, seed=seed)[0] for e in engines]
        ref_obs = obs0[0]
        for e, o in zip(engines[1:], obs0[1:]):
            o = torch.from_numpy(o).to(dev) if e.host else o
            assert torch.equal(_bits(ref_obs), _bits(o)), f"{e.name}: reset obs"
        h = ref_obs.cpu().numpy()
        for lo, ro in zip(windows.los, windows.reset(seed)):
            assert np.array_equal(h[lo:lo + m], ro), f"window {lo}: reset obs"
        if force is not None:
            _force_falls(engines, windows, *force)
            pool = [np.zeros(n, dtype=np.int64)]
        else:
            rng = np.random.default_rng(1234)
            pool = [_random_actions(env_id, n, rng) for _ in range(8)]
        pool_dev = [torch.as_tensor(a, device=dev) for a in pool]
        with concurrent.futures.ThreadPoolExecutor(max_workers=1) as oracle_thread:
            for t in range(steps):
                a_h, a_d = pool[t % len(pool)], pool_dev[t % len(pool)]
                refs = oracle_thread.submit(windows.step, a_h)   # the oracle steps while the GPU does
                outs = [e.step(a_d, a_h) for e in engines]
                for e, out in zip(engines[1:], outs[1:]):
                    _assert_same(outs[0], out, f"step {t}, {e.name}")
                parked, resets = (int(x[0]) for x in engines[0].counts())
                steps_counts.append((parked, resets))
                for e in engines[1:]:
                    p, r = e.counts()
                    assert int(p.sum()) == (parked if e.toi_deferred else 0), f"step {t}, {e.name}: parked envs"
                    assert int(r.sum()) == (resets if e.reset_deferred else 0), f"step {t}, {e.name}: resets"
                    if e.host:
                        np.maximum(chunk_max[e.name][0], p, out=chunk_max[e.name][0])
                        np.maximum(chunk_max[e.name][1], r, out=chunk_max[e.name][1])
                windows.check(tuple(x.cpu().numpy() for x in outs[0]), refs.result(), f"step {t}")
        _report(case, n, steps_counts, chunk_max)
        snap0 = engines[0].env.snapshot()
        diffs = {e.name: _snapshot_words_differ(snap0, e.call(e.env.snapshot)) for e in engines[1:]}
        assert not any(diffs.values()), f"snapshot words that differ from the default's, word: rows: {diffs}"
    finally:
        for e in engines:
            e.env.close()
        windows.close()
    return steps_counts, chunk_max


def _report(case, n, steps_counts, chunk_max):
    """The counts the docstrings quote (pytest -rP shows them)."""
    sms = _sms()
    grid = min(n, TOI_CTAS_PER_SM * sms)
    p = max(c[0] for c in steps_counts)
    r = max(c[1] for c in steps_counts)
    line = (f"{case}: {sms} SMs, TOI grid {grid}: largest parked {p} (L = {_lanes(p, grid)}), largest resets {r} "
            f"({RESET_CTAS_PER_SM * sms * RESET_THREADS} reset-list threads)")
    for name, (cp, cr) in chunk_max.items():
        line += f"; {name}: largest parked per chunk {cp.max()} (L = {_lanes(int(cp.max()), min(n // len(cp), grid))})"
    print(line)


def _assert_multi_lane(n, steps_counts):
    """some step parks more envs than the TOI grid has warps: L >= 2"""
    grid = min(n, TOI_CTAS_PER_SM * _sms())
    assert max(c[0] for c in steps_counts) > grid


def _assert_second_round(n, steps_counts):
    """some step parks more than 32 envs per TOI warp: L = 32 and a second round"""
    grid = min(n, TOI_CTAS_PER_SM * _sms())
    assert max(c[0] for c in steps_counts) > 32 * grid


def _assert_all_slots_used(chunk_max):
    """every counter slot of the 64-chunk host path counted parked envs in some step"""
    parked, _ = chunk_max["host_64"]
    assert len(parked) == 64 and bool((parked > 0).all())


def test_bench_lunar():
    """LunarLander-v2 as bench.py times it: 2^16 envs, 250 warm-up steps of random play, then 60 more.  On an H100
    (132 SMs, TOI grid 1 584): up to 3 739 envs parked in a step (L = 3), up to 1 343 resets; at most 802 parked in a
    chunk of five and 84 in a chunk of 64."""
    n = 1 << 16
    counts, chunks = _run("bench_lunar", "LunarLander-v2", n, WARMUP + 60, m=4096, host64=True)
    _assert_multi_lane(n, counts)
    _assert_all_slots_used(chunks)


def test_continuous_lunar():
    """LunarLanderContinuous-v2: 2^16 envs, 250 + 40 steps of random play.  On an H100: up to 3 102 envs parked in a
    step (L = 2), up to 1 216 resets."""
    n = 1 << 16
    counts, chunks = _run("continuous_lunar", "LunarLanderContinuous-v2", n, WARMUP + 40, m=4096)
    _assert_multi_lane(n, counts)


def test_bench_walker():
    """BipedalWalker-v3 as bench.py times it: 2^16 envs, 250 warm-up steps of random play, then 40 more.  On an H100:
    all 65 536 envs parked in a step (L = 32, two rounds), up to 768 resets; 13 312 parked in a chunk of five (L = 9)
    and 1 024 in a chunk of 64."""
    n = 1 << 16
    counts, chunks = _run("bench_walker", "BipedalWalker-v3", n, WARMUP + 40, m=2048, host64=True)
    _assert_second_round(n, counts)
    _assert_all_slots_used(chunks)


def test_hardcore_ragged():
    """BipedalWalkerHardcore-v3 at 2^16 + 77 envs: the step kernel's last CTA and the last host chunk are partial.
    On an H100: all 65 613 envs parked in a step (L = 32, two rounds), up to 785 resets; 13 312 parked in a chunk of
    five (L = 9)."""
    n = (1 << 16) + 77
    counts, chunks = _run("hardcore_ragged", "BipedalWalkerHardcore-v3", n, WARMUP + 40, m=2048)
    _assert_second_round(n, counts)


def test_walker_whole_batch_truncation():
    """BipedalWalker-v3 at 2^16 envs with a TimeLimit of 20 steps: every env still standing truncates at steps 20
    and 40, all in the same step and while most are parked.  On an H100: 65 536 resets in one step, every env parked
    in one step."""
    n = 1 << 16
    counts, chunks = _run("walker_whole_batch_truncation", "BipedalWalker-v3", n, 45, m=2048, max_episode_steps=20)
    sms = _sms()
    lim = RESET_CTAS_PER_SM * sms * RESET_THREADS
    trunc = [c for c in counts if c[1] > lim]
    assert trunc, "a step with more resets than the reset-list kernel has threads"
    assert all(c[0] > 0 for c in trunc), "... with envs parked in the same step"


FALL_VY = -95.0   # below Box2D's translation clamp (2 m per step), as in test_oracle_box2d.py


@pytest.mark.parametrize("pattern", ["all", "every_4th"])
def test_forced_toi_lunar(pattern):
    """LunarLander-v2 at 2^16 envs: right after reset, the pattern's landers are thrown down at 95 m/s (all three
    bodies, in the engines' snapshot rows and in the oracles alike) and every env steps with action 0 until they
    have hit the pad.  "all": every env parks in the same step, more than 32 per TOI warp, and more envs reset at
    once than the reset-list kernel has threads.  "every_4th": every TOI warp gets between 2 and 32 lanes.  On an
    H100: 65 536 parked and 65 536 resets in one step ("all"), 16 384 parked (L = 11) and 16 384 resets
    ("every_4th")."""
    n = 1 << 16
    mask = np.ones(n, dtype=bool) if pattern == "all" else np.arange(n) % 4 == 0
    counts, chunks = _run(f"forced_toi_lunar[{pattern}]", "LunarLander-v2", n, 12, m=4096, force=(mask, FALL_VY),
                          seed=3)
    sms = _sms()
    grid = min(n, TOI_CTAS_PER_SM * sms)
    if pattern == "all":
        _assert_second_round(n, counts)
        assert max(c[1] for c in counts) > RESET_CTAS_PER_SM * sms * RESET_THREADS
    else:
        assert any(grid < c[0] <= 32 * grid for c in counts)
