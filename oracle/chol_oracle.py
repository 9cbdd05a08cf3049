"""Reference for dense symmetric solves A x = b that does not share a factorisation's rounding: the exactly rounded
residual b - A x (Dekker's TwoProduct of every term, Veltkamp's split, then math.fsum per row) and iterative refinement
on it.  Used to judge the reduced-system Cholesky solve of the Gauss-Newton step (tests/test_gpu_chol.py).

Refinement runs in the diagonal scaling by powers of two (exact: A_s = S A S, b_s = S b, x = S x_s), so its rate is set
by the condition number of the diagonally scaled matrix, which is what the rows of a bundle-adjustment system need
(pose rows against bias rows differ by 1e12 in their diagonal).  Each round contracts the error by about kappa_s * eps;
four rounds reach the correctly rounded solution up to an ulp for kappa_s up to ~1e13."""
import math

import numpy as np

_SPLITTER = 134217729.0            # 2^27 + 1: Veltkamp's split of a double into two 26-bit halves


def _split(a):
    c = _SPLITTER * a
    hi = c - (c - a)
    return hi, a - hi


def two_product(a, b):
    """p, e with p = fl(a b) and p + e = a b exactly (no overflow / underflow), elementwise"""
    p = a * b
    ah, al = _split(a)
    bh, bl = _split(b)
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def exact_residual(A, x, b):
    """b - A x, each entry the exactly rounded value of the exact sum"""
    A, x, b = np.asarray(A, float), np.asarray(x, float), np.asarray(b, float)
    P, E = two_product(A, x[None, :])
    terms = np.concatenate([b[:, None], -P, -E], axis=1)
    return np.array([math.fsum(row) for row in terms.tolist()])


def pow2_scaling(A):
    """powers of two s_i ~ 1 / sqrt(A_ii) (1 where the diagonal is not positive and finite)"""
    d = np.diag(np.asarray(A, float))
    ok = np.isfinite(d) & (d > 0)
    e = np.zeros(len(d))
    e[ok] = np.round(-0.5 * np.log2(d[ok]))
    return np.ldexp(1.0, e.astype(int))


def refined_solve(A, b, rounds=4):
    """x with A x = b to about an ulp: np.linalg.solve, then `rounds` corrections by the exact residual, all in the
    power-of-two diagonal scaling"""
    A, b = np.asarray(A, float), np.asarray(b, float)
    s = pow2_scaling(A)
    As, bs = A * s[:, None] * s[None, :], b * s
    x = np.linalg.solve(As, bs)
    for _ in range(rounds):
        x = x + np.linalg.solve(As, exact_residual(As, x, bs))
    return x * s


def _two_sum(a, b):
    """s, e with s = fl(a + b) and s + e = a + b exactly (Knuth), elementwise"""
    s = a + b
    z = s - a
    return s, (a - (s - z)) + (b - z)


def dd_identity_residual(A, X):
    """I - A X for square A, X, every entry summed in double-double (Ogita, Rump and Oishi's Sum2 over the exact
    products of TwoProduct): as accurate as a sum in twice the working precision, then rounded"""
    n = A.shape[0]
    s, c = np.eye(n), np.zeros((n, n))
    for k in range(n):
        p, pe = two_product(A[:, k:k + 1], X[k:k + 1, :])
        s, t = _two_sum(s, -p)
        c -= pe
        c += t
    return s + c


def refined_inverse(A, rounds=4):
    """A^-1 of a symmetric positive definite A by refinement as refined_solve does it (in the power-of-two diagonal
    scaling A_s = S A S, A^-1 = S A_s^-1 S exactly), for all columns at once, with the residual I - A_s Y in
    double-double (dd_identity_residual) in place of the exactly rounded one"""
    A = np.asarray(A, float)
    if A.shape[0] == 0:
        return np.zeros((0, 0))
    s = pow2_scaling(A)
    As = A * s[:, None] * s[None, :]
    Y = np.linalg.solve(As, np.eye(len(s)))
    for _ in range(rounds):
        Y = Y + np.linalg.solve(As, dd_identity_residual(As, Y))
    return Y * s[:, None] * s[None, :]


def backward_error(A, x, b):
    """componentwise backward error max_i |b - A x|_i / (|A| |x| + |b|)_i with the exactly rounded residual"""
    A, x, b = np.asarray(A, float), np.asarray(x, float), np.asarray(b, float)
    r = np.abs(exact_residual(A, x, b))
    den = np.abs(A) @ np.abs(x) + np.abs(b)
    with np.errstate(invalid="ignore", divide="ignore"):
        q = np.where(r == 0.0, 0.0, r / den)
    return float(np.max(q)) if len(q) else 0.0


def scaled_condition(A):
    """kappa_2 of D^-1/2 A D^-1/2, D = diag(A) (the matrix's condition number in the diagonal scaling)"""
    d = np.sqrt(np.diag(A))
    return float(np.linalg.cond(A / np.outer(d, d)))


def scaled_forward_error(x, x_ref, A):
    """max_i |x - x_ref|_i sqrt(A_ii) / max_i |x_ref|_i sqrt(A_ii)"""
    d = np.sqrt(np.diag(A))
    den = np.max(np.abs(x_ref * d))
    return float(np.max(np.abs((x - x_ref) * d)) / den) if den > 0 else float(np.max(np.abs(x)))
