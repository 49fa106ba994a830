"""An annealed update horizon: BBF's schedule of the multi-step n and the discount gamma after every reset.

Update u of a cycle (u = learn() calls since the Agent was built or since its last reset_parameters()) trains with

    f   = min(u, T) / T                                                      (float64)
    n_u = round_half_even(exp(log n0 + f (log n1 - log n0)))
    g_u = 1 - exp(log(1 - g0) + f (log(1 - g1) - log(1 - g0)))

with exact ends (f = 0 gives (n0, g0), f = 1 gives (n1, g1)) and a start equal to its end held constant.  BBF (Schwarzer
et al. 2023) uses T = 10 000, n 10 -> 3, gamma 0.97 -> 0.997.

The T + 1 rows (rb_horizon of include/rainbow_b200.h) are built here in Python's float64 arithmetic, once, and uploaded.
rb_horizon_advance copies row min(counter, T) into a fixed `current` row and advances the device counter; the gather reads
that row (rb_gather_horizon).  Nothing on the host is frozen into a captured update graph, and `step` mirrors the device
counter without a synchronisation.
"""
import math

import numpy as np
import torch

from . import _lib

MAX_ANNEAL_STEPS = 65536   # RB_MAX_ANNEAL_STEPS
MAX_WINDOW = 64            # RB_MAX_WINDOW
ROW_DTYPE = np.dtype([("n", "<i4"), ("gamma_n", "<f4"), ("gamma_pow", "<f4", (MAX_WINDOW,))])


def _int_option(v, name):
    if isinstance(v, bool) or isinstance(v, float) and not v.is_integer() or int(v) != v:
        raise ValueError(f"{name} must be an integer, got {v!r}")
    return int(v)


def horizon_options(args):
    """(T, n0, n1, g0, g1) from `args`, checked, or None when args.anneal_steps is 0 / absent.  n1 = args.multi_step and
    g1 = args.discount; args.multi_step_start and args.discount_start default to them.  ValueError for T outside
    [1, MAX_ANNEAL_STEPS], n0 < 1, a gamma outside [0, 1] or not finite, an annealed gamma (g0 != g1) with an end at 1, and
    either start given while annealing is off and different from its end."""
    T = getattr(args, "anneal_steps", None)
    T = 0 if T is None else _int_option(T, "anneal_steps")
    n1, g1 = _int_option(args.multi_step, "multi_step"), float(args.discount)
    n0 = getattr(args, "multi_step_start", None)
    n0 = n1 if n0 is None else _int_option(n0, "multi_step_start")
    g0 = getattr(args, "discount_start", None)
    g0 = g1 if g0 is None else float(g0)
    if T == 0:
        if (n0, g0) != (n1, g1):
            raise ValueError("multi_step_start / discount_start need args.anneal_steps > 0")
        return None
    if not 1 <= T <= MAX_ANNEAL_STEPS:
        raise ValueError(f"anneal_steps must be 0 or in [1, {MAX_ANNEAL_STEPS}], got {T}")
    if n0 < 1 or n1 < 1:
        raise ValueError(f"multi_step_start and multi_step must be >= 1, got {n0} and {n1}")
    for name, g in (("discount_start", g0), ("discount", g1)):
        if not (math.isfinite(g) and 0.0 <= g <= 1.0):
            raise ValueError(f"{name} must be in [0, 1], got {g}")
    if g0 != g1 and max(g0, g1) >= 1.0:
        raise ValueError(f"annealing the discount needs both ends below 1, got {g0} -> {g1}")
    return T, n0, n1, g0, g1


def horizon_at(u, T, n0, n1, g0, g1):
    """(n_u, gamma_u) of update u, in Python float64 (module docstring)."""
    f = min(max(int(u), 0), T) / T
    if f == 0.0:
        return n0, g0
    if f == 1.0:
        return n1, g1
    n = n0 if n0 == n1 else round(math.exp(math.log(n0) + f * (math.log(n1) - math.log(n0))))
    g = g0 if g0 == g1 else 1.0 - math.exp(math.log(1.0 - g0) + f * (math.log(1.0 - g1) - math.log(1.0 - g0)))
    return int(n), g


def horizon_table(T, n0, n1, g0, g1):
    """numpy ROW_DTYPE [T + 1]: row u holds n_u, fl32(g_u ** n_u) and fl32(g_u ** k) for k < n_u (zeros beyond), the
    powers in Python doubles like memory.py:101."""
    rows = np.zeros(T + 1, dtype=ROW_DTYPE)
    for u in range(T + 1):
        n, g = horizon_at(u, T, n0, n1, g0, g1)
        rows["n"][u] = n
        rows["gamma_n"][u] = np.float32(g ** n)
        rows["gamma_pow"][u, :n] = np.array([g ** k for k in range(n)], dtype=np.float64).astype(np.float32)
    return rows


class HorizonSchedule:
    """The schedule's host table and its device side: the table, the int64 step counter and the current row."""

    def __init__(self, T, n0, n1, g0, g1, device):
        self.T, self.n0, self.n1, self.g0, self.g1 = int(T), int(n0), int(n1), float(g0), float(g1)
        self.n_max = max(self.n0, self.n1)
        if self.n_max > MAX_WINDOW:
            raise ValueError(f"multi-step horizon {self.n_max} exceeds {MAX_WINDOW}")
        self.device = torch.device(device)
        self.rows = horizon_table(self.T, self.n0, self.n1, self.g0, self.g1)
        self.table = torch.from_numpy(self.rows.view(np.uint8).copy()).to(self.device)
        self.counter = torch.zeros(1, dtype=torch.int64, device=self.device)
        self.current = torch.zeros(ROW_DTYPE.itemsize, dtype=torch.uint8, device=self.device)
        self.step = 0          # host mirror of `counter`: the cycle step of the next update
        self._stream = None
        self._lib = _lib.load()

    @classmethod
    def from_args(cls, args, device):
        opts = horizon_options(args)
        return None if opts is None else cls(*opts, device)

    def at(self, u):
        """(n_u, gamma_u) of cycle step u."""
        return horizon_at(u, self.T, self.n0, self.n1, self.g0, self.g1)

    def side_stream(self):
        if self._stream is None:
            self._stream = torch.cuda.Stream(device=self.device)
        return self._stream

    def advance(self):
        """rb_horizon_advance on the current stream (graph capturable): current <- row min(counter, T), counter + 1.  The
        host mirror follows unless a graph is being captured; whoever replays the graph counts the replays."""
        _lib.check(self._lib.rb_horizon_advance(_lib.ptr(self.table), self.T, _lib.ptr(self.counter),
                                                _lib.ptr(self.current), _lib.stream()))
        if not torch.cuda.is_current_stream_capturing():
            self.step += 1

    def restart(self):
        """Back to u = 0 (host mirror and device counter), on the current stream; not inside a graph capture."""
        self.set_step(0)

    def set_step(self, u):
        self.counter.fill_(int(u))
        self.step = int(u)
