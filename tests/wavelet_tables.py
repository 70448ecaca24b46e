"""Symlet (sym4-sym20) and coiflet (coif3-coif6) decomposition low-pass filters from their defining equations, at 60 digits.

Run as a script, it prints the float64 tables that aphantasia_b200/_wavelets.py holds as literals; tests/test_wavelets_host.py
recomputes them and compares. Every filter is returned in PyWavelets' dec_lo order (rec_lo is its reverse), summing to sqrt(2).

Symlets (`symlet_dec_lo`). The Daubechies-N polynomial P(y) = sum_k C(N-1+k, k) y^k, y = sin^2(w/2), has N-1 roots; each
root y gives a reciprocal pair z, 1/z of z^2 - (2 - 4y) z + 1, and conjugate roots y give conjugate pairs. A root set takes
one member of every pair, together with N zeros at z = -1 (exactly as the minimum-phase `_daubechies_rec_lo`, which takes
every root inside the unit circle). Grouping conjugates, there are 2^G real filters. Least-asymmetric rule:
  * The phase of m0(w) = sum_k rec_lo[k] e^{-ikw} is linear plus Phi(w) = sum_g s_g phi_g(w), where phi_g(w) =
    sum_{r in g} arg(1 - r e^{-iw}) over the inside roots r of group g, and s_g = +1 when the set takes them, -1 when it
    takes their reciprocals. Phi(0) = Phi(pi) = 0. Its sine series is Phi(w) = sum_n a_n sin(nw), a_n = sum_g s_g
    Re(sum_{r in g} r^n) / n, so integral_0^pi Phi^2 dw = (pi / 2) sum_n a_n^2.
  * Take the root set with the least integral of Phi^2: the phase closest to linear in the least-squares sense.
  * A set and its reflection (every s_g negated: the time-reversed filter) tie. Take the one that keeps the group nearest
    the positive real axis (smallest |arg z|) inside the unit circle; that group is the only one for N = 2 and 3, so sym2 /
    sym3 are db2 / db3.

Coiflets (`coiflet_dec_lo`). coifN has L = 6N taps h[0..L-1] with
  * sum_k h[k] = sqrt(2) and sum_k h[k] h[k + 2m] = delta_m for m = 0 .. 3N-1 (orthonormal even shifts),
  * sum_k (-1)^k k^p h[k] = 0 for p = 0 .. 2N-1 (2N vanishing wavelet moments; rec_hi[k] = (-1)^k h[k]),
  * sum_k (k - c)^p h[k] = 0 for p = 1 .. 2N-1 about c = 4N - 1 (2N-1 vanishing scaling moments).
These 7N equations in 6N unknowns have several real solutions. Selection rule: Levenberg-Marquardt in float64 started from
the symmetric Lagrange (Deslauriers-Dubuc) half-band filter with the same moments, h[c] = 1/sqrt(2) and h[c + j] for odd
|j| < 2N the Lagrange weights of the nodes c +- 1, c +- 3, .. at c, divided by sqrt(2); that is the interpolating filter the
coiflets approximate. Gauss-Newton then refines that solution to 60 digits. This reproduces the published coif1 and coif2
(to their own accuracy: their even shifts are orthonormal to 9e-13 and 1e-11 only) and the published coif3's end taps.
"""
import itertools
import math
from math import comb

import mpmath as mp
import numpy as np

DPS = 60


def _polyfrom(roots):
    c = [mp.mpc(1)]
    for r in roots:
        c = [a - r * b for a, b in zip(c + [0], [0] + c)]
    return [mp.re(x) for x in c]


def _normalised(h):
    s = mp.fsum(h)
    return [x / s * mp.sqrt(2) for x in h]


def symlet_dec_lo(N):
    """symN dec_lo, N >= 2, as 60-digit mpf values"""
    with mp.workdps(DPS):
        ys = mp.polyroots([comb(N - 1 + k, k) for k in range(N)][::-1], maxsteps=500, extraprec=4 * DPS)
        tiny = mp.mpf(10) ** (-DPS // 2)
        groups = []                                     # inside roots of each conjugate group
        for y in ys:
            if mp.im(y) < -tiny:
                continue
            a = 2 - 4 * y
            z = (a + mp.sqrt(a * a - 4)) / 2
            z = 1 / z if abs(z) > 1 else z
            groups.append([mp.re(z)] if abs(mp.im(y)) < tiny else [z, mp.conj(z)])
        groups.sort(key=lambda g: abs(mp.arg(g[0])))
        n = np.arange(1, 64 * N + 1)
        a = np.array([[float(mp.re(sum(r ** k for r in g))) for k in n] for g in groups]) / n
        best = min((float(np.sum((np.array((1,) + s) @ a) ** 2)), s) for s in itertools.product((1, -1), repeat=len(groups) - 1))[1]
        roots = [-1] * N
        for g, s in zip(groups, (1,) + best):
            roots += g if s > 0 else [1 / r for r in g]
        return _normalised(_polyfrom(roots))[::-1]


def lagrange_halfband(N):
    """the symmetric interpolating half-band filter with 2N vanishing moments, on coifN's 6N taps centred at 4N - 1"""
    L, c = 6 * N, 4 * N - 1
    h = np.zeros(L)
    h[c] = 1.
    nodes = [2 * j + 1 for j in range(-N, N)]
    for x in nodes:
        h[c + x] = math.prod(-y / (x - y) for y in nodes if y != x)
    return h / math.sqrt(2)


def coiflet_equations(h, N):
    """(residuals F, Jacobian rows J) of coifN's defining equations at h; the moments use x = (k - c) / 2N"""
    L, c = 6 * N, 4 * N - 1
    one = mp.mpf(1) if isinstance(h[0], mp.mpf) else 1.
    x = [(k - c) * one / (2 * N) for k in range(L)]
    F, J = [sum(h) - one * (mp.sqrt(2) if isinstance(one, mp.mpf) else math.sqrt(2))], [[one] * L]
    for m in range(3 * N):
        F.append(sum(h[k] * h[k + 2 * m] for k in range(L - 2 * m)) - (one if m == 0 else 0))
        J.append([(h[j + 2 * m] if j + 2 * m < L else 0) + (h[j - 2 * m] if j >= 2 * m else 0) for j in range(L)])
    rows = [[(-1) ** k * x[k] ** p for k in range(L)] for p in range(2 * N)] + [[x[k] ** p for k in range(L)] for p in range(1, 2 * N)]
    for row in rows:
        J.append(row)
        F.append(sum(r * v for r, v in zip(row, h)))
    return F, J


def coiflet_dec_lo(N):
    """coifN dec_lo, N >= 1, as 60-digit mpf values"""
    from scipy.optimize import least_squares

    def fj(h):
        F, J = coiflet_equations(list(h), N)
        return np.array(F, dtype=np.float64), np.array(J, dtype=np.float64)
    h0 = least_squares(lambda h: fj(h)[0], lagrange_halfband(N), jac=lambda h: fj(h)[1], method='lm',
                       xtol=1e-15, ftol=1e-15, gtol=1e-15).x
    with mp.workdps(DPS):
        h = [mp.mpf(float(v)) for v in h0]
        for _ in range(12):
            F, J = coiflet_equations(h, N)
            if max(abs(f) for f in F) < mp.mpf(10) ** (5 - DPS):
                return h
            Jm = mp.matrix(J)
            dx = mp.lu_solve(Jm.T * Jm, Jm.T * mp.matrix(F))
            h = [a - d for a, d in zip(h, dx)]
    raise RuntimeError('coif%d: Gauss-Newton did not converge' % N)


SYMLETS = range(4, 21)
COIFLETS = range(3, 7)


def _literal(name, tables):
    lines = ['%s = {' % name]
    for n, h in tables.items():
        vals = [repr(float(v)) for v in h]
        rows, row = [], []
        for v in vals:
            if row and len(', '.join(row + [v])) > 112:
                rows.append(', '.join(row))
                row = []
            row.append(v)
        rows.append(', '.join(row))
        lines.append('    %d: [%s],' % (n, (',\n' + ' ' * 8).join(rows)))
    return '\n'.join(lines + ['}'])


if __name__ == '__main__':
    print(_literal('SYM_DEC_LO', {n: symlet_dec_lo(n) for n in SYMLETS}))
    print(_literal('COIF_DEC_LO', {n: coiflet_dec_lo(n) for n in COIFLETS}))
