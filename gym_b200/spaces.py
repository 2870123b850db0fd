"""The three space types the in-scope environments use, plus ``batch_space``.

Host-side objects only (they describe the tensors; they are not on the hot
path).  Behaviour follows the reference so that agent code reading
``envs.single_action_space.n``, calling ``envs.action_space.sample()`` after
``.seed(s)`` or testing ``x in space`` sees the same results:

* ``Space``          gym/spaces/space.py:24-150
* ``Box``            gym/spaces/box.py:53-238
* ``Discrete``       gym/spaces/discrete.py:20-94
* ``MultiDiscrete``  gym/spaces/multi_discrete.py:40-123
* ``batch_space``    gym/vector/utils/spaces.py:17-68

Dict/Tuple/Graph/Sequence/Text spaces are out of scope (no in-scope env uses them).
"""
from copy import deepcopy

import numpy as np

from gym_b200 import error


def np_random(seed=None):
    """gym/utils/seeding.py:9-27 -> (Generator(PCG64(SeedSequence(seed))), entropy)."""
    if seed is not None and not (isinstance(seed, (int, np.integer)) and 0 <= seed):
        raise error.Error(f"Seed must be a non-negative integer or omitted, not {seed}")
    seed_seq = np.random.SeedSequence(None if seed is None else int(seed))
    return np.random.Generator(np.random.PCG64(seed_seq)), seed_seq.entropy


class Space:
    """Base class: shape, dtype and a lazily seeded private Generator."""

    def __init__(self, shape=None, dtype=None, seed=None):
        self._shape = None if shape is None else tuple(shape)
        self.dtype = None if dtype is None else np.dtype(dtype)
        self._np_random = None
        if seed is not None:
            if isinstance(seed, np.random.Generator):
                self._np_random = seed
            else:
                self.seed(seed)

    @property
    def np_random(self):
        if self._np_random is None:
            self.seed()
        return self._np_random

    @property
    def shape(self):
        return self._shape

    def seed(self, seed=None):
        self._np_random, seed = np_random(seed)
        return [seed]

    def sample(self, mask=None):
        raise NotImplementedError

    def contains(self, x):
        raise NotImplementedError

    def __contains__(self, x):
        return self.contains(x)


def _is_number(x):
    return np.issubdtype(type(x), np.integer) or np.issubdtype(type(x), np.floating)


def _full(value, dtype, shape, inf_sign):
    """Scalar or array bound -> array of `dtype`; +-inf becomes the dtype's extreme for ints."""
    dtype = np.dtype(dtype)
    if _is_number(value):
        if np.isinf(value) and dtype.kind != "f":
            info = np.iinfo(dtype)
            value = info.max if inf_sign == "+" else info.min
        return np.full(shape, value, dtype=dtype)
    arr = np.asarray(value)
    if dtype.kind != "f" and np.any(np.isinf(arr)):
        info = np.iinfo(dtype)
        arr = arr.astype(np.float64)
        arr = np.where(np.isposinf(arr), info.max, np.where(np.isneginf(arr), info.min, arr))
    return arr.astype(dtype)


class Box(Space):
    """Closed box in R^n (gym/spaces/box.py:53-134)."""

    def __init__(self, low, high, shape=None, dtype=np.float32, seed=None):
        assert dtype is not None, "Box dtype must be explicitly provided, cannot be None."
        self.dtype = np.dtype(dtype)
        if shape is not None:
            shape = tuple(int(d) for d in shape)
        elif isinstance(low, np.ndarray):
            shape = low.shape
        elif isinstance(high, np.ndarray):
            shape = high.shape
        elif _is_number(low) and _is_number(high):
            shape = (1,)
        else:
            raise ValueError("Box shape is inferred from low and high: give np.ndarray bounds or a shape")
        _low = np.full(shape, low, dtype=float) if _is_number(low) else np.asarray(low)
        _high = np.full(shape, high, dtype=float) if _is_number(high) else np.asarray(high)
        self.bounded_below = -np.inf < _low
        self.bounded_above = np.inf > _high
        self.low = _full(low, self.dtype, shape, "-")
        self.high = _full(high, self.dtype, shape, "+")
        assert self.low.shape == shape and self.high.shape == shape, "low/high do not match the shape"
        super().__init__(shape, self.dtype, seed)

    def is_bounded(self, manner="both"):
        below, above = bool(np.all(self.bounded_below)), bool(np.all(self.bounded_above))
        if manner == "both":
            return below and above
        if manner == "below":
            return below
        if manner == "above":
            return above
        raise ValueError(f"manner is not in {{'below', 'above', 'both'}}, actual value: {manner}")

    def sample(self, mask=None):
        """gym/spaces/box.py:171-222: uniform / shifted exponential / normal per coordinate."""
        if mask is not None:
            raise error.Error(f"Box.sample cannot be provided a mask, actual value: {mask}")
        high = self.high if self.dtype.kind == "f" else self.high.astype("int64") + 1
        sample = np.empty(self.shape)
        unbounded = ~self.bounded_below & ~self.bounded_above
        upp_bounded = ~self.bounded_below & self.bounded_above
        low_bounded = self.bounded_below & ~self.bounded_above
        bounded = self.bounded_below & self.bounded_above
        sample[unbounded] = self.np_random.normal(size=unbounded[unbounded].shape)
        sample[low_bounded] = (self.np_random.exponential(size=low_bounded[low_bounded].shape)
                               + self.low[low_bounded])
        sample[upp_bounded] = (-self.np_random.exponential(size=upp_bounded[upp_bounded].shape)
                               + self.high[upp_bounded])
        sample[bounded] = self.np_random.uniform(low=self.low[bounded], high=high[bounded],
                                                 size=bounded[bounded].shape)
        if self.dtype.kind == "i":
            sample = np.floor(sample)
        return sample.astype(self.dtype)

    def contains(self, x):
        if not isinstance(x, np.ndarray):
            try:
                x = np.asarray(x, dtype=self.dtype)
            except (ValueError, TypeError):
                return False
        return bool(np.can_cast(x.dtype, self.dtype) and x.shape == self.shape
                    and np.all(x >= self.low) and np.all(x <= self.high))

    def __repr__(self):
        def short(a):
            return str(a.flat[0]) if a.size and np.min(a) == np.max(a) else str(a)
        return f"Box({short(self.low)}, {short(self.high)}, {self.shape}, {self.dtype})"

    def __eq__(self, other):
        return (isinstance(other, Box) and self.shape == other.shape
                and np.allclose(self.low, other.low) and np.allclose(self.high, other.high))


class Discrete(Space):
    """{start, ..., start+n-1} (gym/spaces/discrete.py:20-40)."""

    def __init__(self, n, seed=None, start=0):
        assert isinstance(n, (int, np.integer)) and n > 0, "n (counts) have to be positive"
        assert isinstance(start, (int, np.integer))
        self.n = int(n)
        self.start = int(start)
        super().__init__((), np.int64, seed)

    def sample(self, mask=None):
        if mask is not None:
            assert isinstance(mask, np.ndarray) and mask.dtype == np.int8 and mask.shape == (self.n,)
            valid = mask == 1
            assert np.all(np.logical_or(mask == 0, valid))
            if np.any(valid):
                return int(self.start + self.np_random.choice(np.where(valid)[0]))
            return self.start
        return int(self.start + self.np_random.integers(self.n))  # discrete.py:81

    def contains(self, x):
        if isinstance(x, int):
            as_int = x
        elif isinstance(x, (np.generic, np.ndarray)) and (np.issubdtype(x.dtype, np.integer) and x.shape == ()):
            as_int = int(x)
        else:
            return False
        return self.start <= as_int < self.start + self.n

    def __repr__(self):
        return f"Discrete({self.n}, start={self.start})" if self.start != 0 else f"Discrete({self.n})"

    def __eq__(self, other):
        return isinstance(other, Discrete) and self.n == other.n and self.start == other.start


class MultiDiscrete(Space):
    """Cartesian product of Discrete spaces (gym/spaces/multi_discrete.py:40-123)."""

    def __init__(self, nvec, dtype=np.int64, seed=None):
        self.nvec = np.array(nvec, dtype=dtype, copy=True)
        assert (self.nvec > 0).all(), "nvec (counts) have to be positive"
        super().__init__(self.nvec.shape, dtype, seed)

    def sample(self, mask=None):
        if mask is not None:
            raise error.Error("MultiDiscrete.sample(mask=...) is not supported by gym_b200")
        return (self.np_random.random(self.nvec.shape) * self.nvec).astype(self.dtype)  # multi_discrete.py:123

    def contains(self, x):
        if isinstance(x, (list, tuple)):
            x = np.array(x)
        return bool(isinstance(x, np.ndarray) and x.shape == self.shape and x.dtype != object
                    and np.can_cast(x.dtype, self.dtype) and np.all(0 <= x) and np.all(x < self.nvec))

    def __repr__(self):
        return f"MultiDiscrete({self.nvec})"

    def __len__(self):
        return self.nvec.shape[0]

    def __eq__(self, other):
        return isinstance(other, MultiDiscrete) and np.all(self.nvec == other.nvec)


PCG64_MULT = 0x2360ED051FC65DA44385DF649FCCF645
_MASK128 = (1 << 128) - 1


def pcg64_jump(state, inc, delta):
    """The PCG64 LCG state ``delta`` draws after ``state`` (PCG's pcg_advance_lcg_128: square-and-multiply over the
    bits of ``delta``, taken mod 2**128 like ``PCG64.advance``)."""
    cur_mult, cur_plus, acc_mult, acc_plus = PCG64_MULT, inc & _MASK128, 1, 0
    delta &= _MASK128
    while delta:
        if delta & 1:
            acc_mult = acc_mult * cur_mult & _MASK128
            acc_plus = (acc_plus * cur_mult + cur_plus) & _MASK128
        cur_plus = (cur_mult + 1) * cur_plus & _MASK128
        cur_mult = cur_mult * cur_mult & _MASK128
        delta >>= 1
    return (acc_mult * state + acc_plus) & _MASK128


def pcg64_state(bit_generator):
    """``bit_generator.state`` of a PCG64 bit generator; ``error.Error`` for any other kind (Philox, PCG64DXSM, ...),
    whose streams the device does not reproduce."""
    state = bit_generator.state
    if state.get("bit_generator") != "PCG64":
        raise error.Error(f"device sampling reproduces numpy's PCG64 stream only; this space's generator is "
                          f"{state.get('bit_generator')}")
    return state


def pcg64_skip(bit_generator, state, count):
    """Move a PCG64 bit generator from ``state`` (as ``pcg64_state`` returned it) to where ``count`` 64-bit draws
    leave it.  The buffered 32-bit draw (``has_uint32`` / ``uinteger``) stays as it was, as the draws of ``random`` /
    ``uniform`` leave it -- ``PCG64.advance`` would clear it."""
    words = state["state"]
    state["state"] = dict(words, state=pcg64_jump(words["state"], words["inc"], count))
    bit_generator.state = state


def batch_space(space, n=1):
    """gym/vector/utils/spaces.py:46-68: Box tiles its bounds, Discrete -> MultiDiscrete([n]*N)."""
    if isinstance(space, Box):
        repeats = tuple([n] + [1] * space.low.ndim)
        return Box(low=np.tile(space.low, repeats), high=np.tile(space.high, repeats),
                   dtype=space.dtype, seed=deepcopy(space.np_random))
    if isinstance(space, Discrete):
        if space.start == 0:
            return MultiDiscrete(np.full((n,), space.n, dtype=space.dtype), dtype=space.dtype,
                                 seed=deepcopy(space.np_random))
        return Box(low=space.start, high=space.start + space.n - 1, shape=(n,), dtype=space.dtype,
                   seed=deepcopy(space.np_random))
    if isinstance(space, MultiDiscrete):
        repeats = tuple([n] + [1] * space.nvec.ndim)
        high = np.tile(space.nvec, repeats) - 1
        return Box(low=np.zeros_like(high), high=high, dtype=space.dtype, seed=deepcopy(space.np_random))
    raise ValueError(f"Cannot batch space with type `{type(space)}`.")
