"""The reference of the reduced-system Cholesky tests (oracle/chol_oracle.py) on its own, without a GPU: its residual
is exactly rounded (against mpmath at 40 digits), and iterative refinement reproduces known integer solutions of integer
SPD systems, plain and scaled by powers of two, up to a condition number of 1e12, to within an ulp."""
import mpmath
import numpy as np
import pytest

from oracle import chol_oracle as co


def _integer_spd(rng, n, m):
    """A = L C L^T with C = B B^T + n I (B integer in [-2, 2]: well conditioned) and L unit lower triangular with a chain
    of m entries -2 below the diagonal (L^-1 holds 2^m: the condition number grows like 4^m); x integer and nonzero (an
    ulp of 0 is no bar), b = A x: all exact in int64 and in double"""
    B = rng.integers(-2, 3, (n, n))
    C = B @ B.T + n * np.eye(n, dtype=np.int64)
    L = np.eye(n, dtype=np.int64)
    for i in range(1, m + 1):
        L[i, i - 1] = -2
    A = L @ C @ L.T
    x = rng.integers(1, 51, n) * rng.choice([-1, 1], n)
    b = A @ x
    assert np.max(np.abs(A)) < 2 ** 52 and np.max(np.abs(b)) < 2 ** 52
    return A.astype(float), x.astype(float), b.astype(float)


def _ulps(x, ref):
    return np.max(np.abs(x - ref) / np.spacing(np.maximum(np.abs(ref), np.finfo(float).tiny)))


def test_exact_residual_is_exactly_rounded():
    rng = np.random.default_rng(11)
    mpmath.mp.dps = 40
    for n in (1, 7, 30):
        for scale in (1.0, 1e-3, 1e8):
            A = rng.standard_normal((n, n)) * scale
            x = np.linalg.solve(A, rng.standard_normal(n))     # so that b - A x cancels to rounding level
            b = A @ x
            r = co.exact_residual(A, x, b)
            for i in range(n):
                ex = mpmath.mpf(b[i]) - mpmath.fsum(mpmath.mpf(A[i, j]) * mpmath.mpf(x[j]) for j in range(n))
                assert r[i] == float(ex), (n, scale, i, r[i], float(ex))


@pytest.mark.parametrize("n,m", [(6, 0), (24, 4), (45, 8), (96, 12), (120, 16), (64, 18)])
def test_refined_solve_reproduces_integer_solutions(n, m):
    rng = np.random.default_rng(n * 100 + m)
    A, x, b = _integer_spd(rng, n, m)
    kappa = np.linalg.cond(A)
    assert kappa < 1e13
    assert _ulps(co.refined_solve(A, b), x) <= 1.0, kappa


def test_refined_solve_reaches_kappa_1e12():
    """the largest condition number the Cholesky tests use"""
    rng = np.random.default_rng(5)
    for n in (40, 96, 160):
        A, x, b = _integer_spd(rng, n, 19)
        kappa = np.linalg.cond(A)
        assert 1e11 <= kappa <= 1e13, kappa
        assert _ulps(co.refined_solve(A, b), x) <= 1.0, kappa


def test_refined_solve_on_scaled_integer_systems():
    """rows and columns scaled by 2^e, e in [-7, 13] (1e-2 ... 1e4, as pose rows against bias rows): the solution is
    x / 2^e, exactly; the unscaled condition number grows by up to 1e12, the scaled one stays that of A"""
    rng = np.random.default_rng(7)
    for n, m in ((30, 4), (60, 10), (90, 16)):
        A, x, b = _integer_spd(rng, n, m)
        s = np.ldexp(1.0, rng.integers(-7, 14, n))
        As, bs, xs = A * np.outer(s, s), b * s, x / s
        assert _ulps(co.refined_solve(As, bs), xs) <= 1.0


def test_backward_error_of_an_exact_solution_is_zero():
    rng = np.random.default_rng(3)
    A, x, b = _integer_spd(rng, 20, 2)
    assert co.backward_error(A, x, b) == 0.0
    x2 = x.copy()
    x2[4] += 1.0
    assert co.backward_error(A, x2, b) > 1e-3
