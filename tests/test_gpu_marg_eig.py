"""The marginaliser's eigen-solver (marg_eig_kernel: Householder tridiagonalisation + implicit QL, the factorisation of
bundle_adjustor.cpp:583-590) through pvio_b200_selftest_eig, against numpy.linalg.eigh of the same stored matrix, at
every size the marginaliser accepts (dk = 15 (N - 1), 15 ... 165) and on the spectra where such solvers go wrong:
graded, repeated, clustered, indefinite, at the 1e-8 clamp, already reduced, with zero rows, and QL's hard case
(Wilkinson W+).  The matrix is stored exactly symmetric, so the kernel (which reads the lower triangle) and eigh factor
the same matrix.

Bars, with u = 2^-53, n = dk and |A| = max |lambda| (normwise backward stability of tridiagonalisation + QL, with a
factor of 64 for the constants; relative accuracy of small eigenvalues of graded matrices is not a property of dense
tridiagonal QL and is not asked for):
  |S^T S - A|_max          <= 64 n u |A| + max |lambda| over the clamped eigenvalues
  |A v - lambda v|         <= 64 n u |A|     per pair (lambda = |S_i|^2, v = S_i / |S_i|)
  |v_i . v_j - delta_ij|   <= 64 n u
  sorted lambda vs eigh    <= 64 n u |A|     (Weyl)
  positive count exact wherever every eigenvalue is further than 1e3 n u |A| from the clamp
  clamped rows of S and their e exactly 0; e_i = v_i . b / sqrt(lambda_i) to 8 n u |b| / sqrt(lambda_i)."""
import numpy as np
import pytest

from pvio_b200 import _lib
from pvio_b200.bundle_adjustor import BundleAdjustor, PvioB200Error

pytestmark = pytest.mark.gpu

U = 2.0 ** -53
CLAMP = 1.0e-8
SIZES = list(range(15, 166, 15))
EINVAL = rf"error {_lib.EINVAL}\b"
BARS = ("recon", "resid", "orth", "weyl", "e")


@pytest.fixture(scope="module")
def ba():
    b = BundleAdjustor(max_windows=1, max_frames=12, max_landmarks=64, max_obs=512)
    yield b
    b.close()


def _sym(A):
    """the matrix the kernel factors: its lower triangle, mirrored"""
    L = np.tril(A)
    return L + np.tril(L, -1).T


def _orth(rng, n):
    Q, R = np.linalg.qr(rng.standard_normal((n, n)))
    return Q * np.sign(np.diag(R))


def _from_spectrum(rng, lam):
    Q = _orth(rng, len(lam))
    return _sym((Q * lam) @ Q.T)


def _ratio(err, bar):
    return 0.0 if err == 0.0 else (err / bar if bar > 0.0 else np.inf)


def _check(A, b, S, e):
    """ratio of each error to its bar (<= 1 passes); asserts the exact properties"""
    n = len(b)
    lam_ref = np.linalg.eigvalsh(A)[::-1]
    nrm = np.max(np.abs(lam_ref))
    tol = 64 * n * U * nrm
    rn = np.linalg.norm(S, axis=1)
    pos = rn > 0
    p = int(pos.sum())
    assert np.all(e[~pos] == 0.0)                           # clamped: the row is 0 (its norm is) and so is its e
    lam = rn[pos] ** 2
    V = S[pos] / rn[pos, None]
    order = np.argsort(-lam)
    lam, V, ep = lam[order], V[order], e[pos][order]
    clamped = np.max(np.abs(lam_ref[p:])) if p < n else 0.0
    r = dict(recon=_ratio(np.max(np.abs(S.T @ S - A)), tol + clamped))
    if p:
        r["resid"] = max(_ratio(x, tol) for x in np.linalg.norm(V @ A - lam[:, None] * V, axis=1))
        r["orth"] = _ratio(np.max(np.abs(V @ V.T - np.eye(p))), 64 * n * U)
        r["weyl"] = _ratio(np.max(np.abs(lam - lam_ref[:p])), tol)
        sq = np.sqrt(lam)
        r["e"] = np.max(np.abs(ep - (V @ b) / sq) / (8 * n * U * np.linalg.norm(b) / sq))
    if np.min(np.abs(lam_ref - CLAMP)) > 1e3 * n * U * nrm:
        assert p == int(np.sum(lam_ref > CLAMP)), (n, p, int(np.sum(lam_ref > CLAMP)))
    return r


def _run(ba, family, problems):
    out = ba.selftest_eig(problems)
    worst = dict.fromkeys(BARS, 0.0)
    for (A, b), (S, e) in zip(problems, out):
        for k, v in _check(A, b, S, e).items():
            assert v <= 1.0, (family, len(b), k, v)
            worst[k] = max(worst[k], v)
    print(f"eigen-solver, {family}: worst error / bar " + ", ".join(f"{k} {v:.2e}" for k, v in worst.items()))
    return out


def _wilkinson_plus(n):
    m = (n - 1) // 2
    return np.diag(np.abs(m - np.arange(n)).astype(float)) + np.diag(np.ones(n - 1), 1) + np.diag(np.ones(n - 1), -1)


def _repeated(rng, n):
    """eigenvalues 7 (multiplicity 30 from n = 30 on), 3 (multiplicity 15), the rest distinct in [1, 1e3]"""
    lam = rng.uniform(1.0, 1e3, n)
    lam[:15] = 3.0
    if n >= 45:
        lam[15:45] = 7.0
    return lam


def _block_zero_rows(rng, n):
    """per 15-frame block a dense SPD block; v / bg / ba (coordinates 6..14) of every other frame have no information, as
    for frames without an IMU factor or prior"""
    A = np.zeros((n, n))
    for f in range(n // 15):
        k = 6 if f % 2 else 15
        s = slice(15 * f, 15 * f + k)
        A[s, s] = _from_spectrum(rng, rng.uniform(1.0, 1e3, k))
    return _sym(A)


def _tridiagonal(rng, n):
    off = rng.uniform(-1.0, 1.0, n - 1)
    off[::9] = 0.0                                            # splits: QL's convergence test sees them at once
    return np.diag(rng.uniform(-10.0, 10.0, n)) + np.diag(off, 1) + np.diag(off, -1)


def _near_clamp(rng, n):
    """|A| = 1, and k eigenvalues at 0.5e-8 / 1.5e-8: either side of the clamp, 5e-9 away"""
    k = max(2, n // 10)
    lam = np.concatenate([[1.0], rng.uniform(0.1, 1.0, n - 1 - k), 1e-8 * (1.0 + 0.5 * (-1.0) ** np.arange(k))])
    return lam


FAMILIES = {
    "spd": lambda rng, n: _from_spectrum(rng, rng.uniform(1.0, 1e3, n)),
    "graded_1e30_1e-4": lambda rng, n: _from_spectrum(rng, np.geomspace(1e30, 1e-4, n)),
    "graded_1e12_1e-12": lambda rng, n: _from_spectrum(rng, np.geomspace(1e12, 1e-12, n)),
    "repeated": lambda rng, n: _from_spectrum(rng, _repeated(rng, n)),
    "block_zero_rows": _block_zero_rows,
    "diagonal": lambda rng, n: np.diag(np.where(np.arange(n) % 7 == 0, 0.0, rng.uniform(-1e3, 1e3, n))),
    "tridiagonal": _tridiagonal,
    "indefinite": lambda rng, n: _from_spectrum(rng, rng.uniform(-1e3, 1e3, n)),
    "near_clamp": lambda rng, n: _from_spectrum(rng, _near_clamp(rng, n)),
    "zero": lambda rng, n: np.zeros((n, n)),
    "1e-9_I": lambda rng, n: 1e-9 * np.eye(n),
    "1e-7_I": lambda rng, n: 1e-7 * np.eye(n),
}


@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_eigen_solver_matches_eigh_at_every_size(ba, family):
    """one launch over all eleven sizes of the family"""
    rng = np.random.default_rng(sorted(FAMILIES).index(family) + 90)
    problems = [(FAMILIES[family](rng, n), rng.standard_normal(n)) for n in SIZES]
    _run(ba, family, problems)


def test_eigen_solver_on_wilkinson_matrices(ba):
    """W+ at the odd sizes: pairs of eigenvalues that agree to many digits, QL's slowest convergence"""
    rng = np.random.default_rng(97)
    _run(ba, "wilkinson", [(_wilkinson_plus(n), rng.standard_normal(n)) for n in SIZES if n % 2])


def test_eigen_solver_on_marginalised_windows(ba):
    """the Hk, bk bo.marginalize leaves for N = 12 windows (dk = 165) with a full prior and with none: the second has a
    null space (yaw and position), whose eigenvalues are rounding noise around the clamp"""
    from oracle import ba_oracle as bo
    from synthetic import synth
    problems = []
    for seed, prior in ((120, "synthetic"), (121, "none")):
        w, st, _ = synth.make_cfg3(N=12, M=120, seed=seed, prior=prior)
        _, _, Hk, bk = bo.marginalize(w, st, index=0)
        problems.append((_sym(Hk), bk))
    _run(ba, "marginalised N = 12", problems)


def test_eigen_solver_does_not_depend_on_its_launch(ba):
    """A matrix factored alone and inside a launch whose largest problem is dk = 165 (more shared memory per CTA), at
    another grid position, gives bit-identical S and e: each CTA's arithmetic depends on its own problem only.  (Every
    size 15 ... 165 fits the 4-slot rotation ring, so both launches pipeline through 4 slots.)"""
    rng = np.random.default_rng(98)
    probs = [(_from_spectrum(rng, rng.uniform(1.0, 1e3, n)), rng.standard_normal(n)) for n in (120, 45)]
    big = (_from_spectrum(rng, rng.uniform(-1e3, 1e3, 165)), rng.standard_normal(165))
    together = ba.selftest_eig([big, probs[1], probs[0]])
    for (A, b), (S, e) in zip(probs, (together[2], together[1])):
        S1, e1 = ba.selftest_eig([(A, b)])[0]
        assert np.array_equal(S, S1) and np.array_equal(e, e1), len(b)


def test_eigen_solver_rejects_sizes_the_marginaliser_does_not_accept(ba):
    for d in (0, 20, 180):
        with pytest.raises(PvioB200Error, match=EINVAL):
            ba.selftest_eig([(np.eye(d), np.ones(d))])
    with pytest.raises(PvioB200Error, match=EINVAL):             # a bad size anywhere rejects the whole call
        ba.selftest_eig([(np.eye(15), np.ones(15)), (np.eye(170), np.ones(170))])
    one = np.zeros(1)
    dk = np.array([15], dtype=np.int32)
    rc = ba.lib.pvio_b200_selftest_eig(ba.h, 0, _lib.ptr(dk), *(_lib.ptr(one) for _ in range(4)))
    assert rc == _lib.EINVAL
