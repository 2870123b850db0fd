"""numpy restatement of the reshaping per-env wrapper chains (FrameStack, TimeAwareObservation, FlattenObservation;
gym_b200/subenv.py, csrc/subenv.cuh) and of the action stages (ClipAction, RescaleAction).  Test infrastructure.

``SubenvShapeRef`` extends ``oracle.subenv_chain.SubenvChainRef`` (whose reward stages it reuses unchanged) with an
observation pipeline that carries the shape and dtype of the observation from stage to stage, letting numpy do the
typing, as the reference wrappers do:

* FrameStack (gym/wrappers/frame_stack.py:164-190): a step appends the new frame, a reset appends it num_stack
  times; the frames keep the dtype they have at that position;
* TimeAwareObservation (time_aware_observation.py:38-71): ``np.append(obs, t)`` flattens and, with t an int64,
  makes the observation float64; t counts the steps since the reset (the terminal row ends in the episode length);
* FlattenObservation (spaces/utils.py:138-141): ``np.asarray(x, dtype=float32).flatten()``;
* NormalizeObservation's batch variance ``(x - x)**2`` is taken in the dtype at its position.
"""
import numpy as np

from oracle.subenv_chain import SubenvChainRef, _update


class SubenvShapeRef(SubenvChainRef):
    """stages: ``[(name, kwargs), ...]`` innermost first; ``obs_dim``: the raw observation's size.  ``step`` / ``reset``
    return flat rows of the chain's output width; ``shape`` is one env's output shape."""

    def __init__(self, stages, env_id, n, obs_dim):
        super().__init__(stages, env_id, n, obs_dim)
        shape, dtype = (self.d,), np.dtype(np.float32)
        self.norm = self.hist = self.t = None
        for name, kw in self.stages:
            if name == "NormalizeObservation":
                w = int(np.prod(shape))
                self.norm = [np.zeros((n, w)), np.ones((n, w)), np.full((n, 1), 1e-4)]
                dtype = np.dtype(np.float64)
            elif name == "FrameStack":
                k = int(kw["num_stack"])
                self.hist = np.zeros((n, k) + shape, dtype)
                shape = (k,) + shape
            elif name == "TimeAwareObservation":
                self.t = np.zeros(n, np.int64)
                shape, dtype = (int(np.prod(shape)) + 1,), np.dtype(np.float64)
            elif name == "FlattenObservation":
                shape, dtype = (int(np.prod(shape)),), np.dtype(np.float32)
        self.shape, self.final_dtype = shape, dtype
        self.normalizes_obs = dtype == np.float64   # the parent's terminal rows take this dtype
        self.width = int(np.prod(shape))
        self.d = self.width
        self._phase, self._done = "reset", None

    def _obs_rows(self, rows, x):
        """The observation stages over the rows `rows` (raw float32 (m, D)) -> flat (m, W) rows in the output dtype.
        The phase says what the rows are: "terminal" (FrameStack appends, t = the step's), "step" (finishing envs:
        their reset row) or "reset"."""
        m = len(rows)
        if self._phase == "reset":
            fill = np.ones(m, bool)
        elif self._phase == "terminal":
            fill = np.zeros(m, bool)
        else:
            fill = self._done[rows]
        tt = None
        if self.t is not None:
            tt = np.where(fill, 0, self.t[rows] + 1).astype(np.int64)
        x = np.asarray(x, np.float32)
        for name, kw in self.stages:
            if name == "NormalizeObservation":
                xf = x.reshape(m, -1)
                mean, var, count = _update(self.norm[0][rows], self.norm[1][rows], self.norm[2][rows], xf,
                                           np.square(xf - xf))
                self.norm[0][rows], self.norm[1][rows], self.norm[2][rows] = mean, var, count
                x = ((xf - mean) / np.sqrt(var + kw["epsilon"])).reshape(x.shape)
            elif name == "ClipObservation":
                x = np.clip(x, kw["low"], kw["high"])
            elif name == "FrameStack":
                h = self.hist[rows]
                assert h.dtype == x.dtype
                h[fill] = x[fill][:, None]
                h[~fill, :-1] = h[~fill, 1:]
                h[~fill, -1] = x[~fill]
                self.hist[rows] = h
                x = h.copy()
            elif name == "TimeAwareObservation":
                x = np.concatenate([x.reshape(m, -1), tt[:, None]], axis=1)
            elif name == "FlattenObservation":
                x = np.asarray(x, np.float32).reshape(m, -1)
        if self.t is not None and self._phase != "terminal":
            self.t[rows] = tt
        if self._phase == "terminal":
            self._phase = "step"
        assert x.dtype == self.final_dtype
        return x.reshape(m, -1)

    def reset(self, obs):
        self._phase = "reset"
        return super().reset(obs)

    def step(self, obs, reward, terminated, truncated, final_obs):
        """As ``SubenvChainRef.step``; the terminal rows are (n, W) in the chain's output dtype."""
        self._done = np.asarray(terminated, bool) | np.asarray(truncated, bool)
        self._phase = "terminal" if self._done.any() else "step"
        return super().step(obs, reward, terminated, truncated, final_obs)


def action_stages(stages, low, high):
    """(op, low, high, min, max) float32 arrays of the action stages in the order they apply (outermost first),
    from the env's action bounds; op "clip" or "rescale".  -> (stages, low, high of the outermost space)."""
    out = []
    low, high = np.asarray(low, np.float32), np.asarray(high, np.float32)
    for name, kw in stages:
        if name == "ClipAction":
            out.insert(0, ("clip", low, high, None, None))
        elif name == "RescaleAction":
            amin = np.zeros(low.shape, np.float32) + np.asarray(kw["min_action"], np.float32)
            amax = np.zeros(low.shape, np.float32) + np.asarray(kw["max_action"], np.float32)
            out.insert(0, ("rescale", low, high, amin, amax))
            low, high = amin, amax
    return out, low, high


def apply_actions(stages, low, high, a):
    """The action the env sees for float32 actions `a` (N, A): clip_action.py:31-40, rescale_action.py:62-82."""
    a = np.asarray(a, np.float32)
    for op, lo, hi, amin, amax in action_stages(stages, low, high)[0]:
        if op == "rescale":
            a = lo + (hi - lo) * ((a - amin) / (amax - amin))
        a = np.clip(a, lo, hi)
        assert a.dtype == np.float32
    return a
