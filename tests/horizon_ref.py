"""An independent float64 reference of the annealed horizon (rainbow_b200.horizon): the schedule written from its
definition with numpy and exact rational rounding, not with the module's own code."""
import math
from fractions import Fraction

import numpy as np


def round_half_even(x):
    """x (a float) to the nearest integer, ties to even, decided on the exact value of the float."""
    q = Fraction(x)
    lo = q.numerator // q.denominator
    rest = q - lo
    if rest > Fraction(1, 2) or (rest == Fraction(1, 2) and lo % 2 == 1):
        return lo + 1
    return lo


def schedule(u, T, n0, n1, g0, g1):
    """(n_u, gamma_u): log-linear in n and in 1 - gamma over f = min(u, T) / T, exact at both ends."""
    if u <= 0:
        return n0, g0
    if u >= T:
        return n1, g1
    f = u / T
    n = n0 if n0 == n1 else round_half_even(math.exp(math.log(n0) + f * (math.log(n1) - math.log(n0))))
    if g0 == g1:
        return int(n), g0
    a, b = math.log(1.0 - g0), math.log(1.0 - g1)
    return int(n), 1.0 - math.exp(a + f * (b - a))


def row(u, T, n0, n1, g0, g1, window=64):
    """(n, gamma_n, gamma_pow[window]) of step u as float32, powers in Python doubles."""
    n, g = schedule(u, T, n0, n1, g0, g1)
    pw = np.zeros(window, np.float32)
    pw[:n] = [np.float32(g ** k) for k in range(n)]
    return n, np.float32(g ** n), pw
