"""The reduced-system Cholesky solve of the Gauss-Newton step (csrc/ba_chol.cuh) judged on its own at fp64 level, against
an exact-residual reference (oracle/chol_oracle.py), through pvio_b200_selftest_chol and through solve_kernel itself.

Modes of the self-test (the variant each production kernel runs for a block count nb = ceil(D / 4)):
  narrow      chol_solve_tiled<false>, 64 threads: the batched visual-only kernel.  It is chosen for systems of at most
              14 free frames (D = 84, nb = 21: solve_smem_one's lean size of 15 free frames passes 48 KB).
  wide        chol_solve<true>, 256 threads: chol_solve_regs<4> for nb <= 41, chol_solve_regs<5> for nb = 42 ... 46 (warp
              0's lanes own two diagonal tiles from nb = 33 on), chol_solve_tiled<true> beyond.
  wide-tiled  chol_solve_tiled<true> forced: the fallback.  Up to nb = 54, the largest packed system within 220 KB.

Bars, fixed from the error analysis of Cholesky (eps = 2^-52, D the number of unknowns):
  componentwise backward error  max_i |b - A x|_i / (|A| |x| + |b|)_i <= 4 D eps   (exactly rounded residual)
  forward error in the diagonal scaling  max |x - x_ref| sqrt(diag A) / max |x_ref| sqrt(diag A) <= 4 D eps kappa_s
with kappa_s the condition number of the diagonally scaled matrix.  A stale or missing tile update breaks the first by
orders of magnitude; no bar is put on the ratio to LAPACK's error, which swings by ~10x at kappa_s = 1e13."""
import functools

import numpy as np
import pytest

from oracle import ba_oracle as bo
from oracle import chol_oracle as co
from synthetic import synth
from pvio_b200 import _lib
from pvio_b200.bundle_adjustor import BundleAdjustor, PvioB200Error

pytestmark = pytest.mark.gpu

EPS = 2.0 ** -52
EINVAL = rf"error {_lib.EINVAL}\b"
NB_MAX = {"narrow": 21, "wide": 46, "wide-tiled": 54}
# D = 6 N (visual windows) and 15 N (inertial ones) that production hands each variant
PROD_D = {"narrow": [6 * k for k in range(1, 15)],
          "wide": [6 * k for k in range(1, 17)] + [15 * k for k in range(1, 12)],
          "wide-tiled": [6 * k for k in range(1, 17)] + [15 * k for k in range(1, 15)]}
KINDS = ("kappa1", "kappa1e4", "kappa1e8", "kappa1e12", "spread", "pinned")


@pytest.fixture(scope="module")
def ba():
    b = BundleAdjustor(max_windows=1, max_frames=16, max_landmarks=320, max_obs=4000)
    yield b
    b.close()


def _spd(rng, D, kappa):
    """unit diagonal, random orthogonal eigenvectors, eigenvalues geometric from 1 to 1 / kappa (before the scaling)"""
    Q, R = np.linalg.qr(rng.standard_normal((D, D)))
    Q = Q * np.sign(np.diag(R))
    M = (Q * np.geomspace(1.0, 1.0 / kappa, D)) @ Q.T
    d = np.sqrt(np.diag(M))
    M = M / np.outer(d, d)
    return 0.5 * (M + M.T)


def _pin(A, b, idx):
    """identity rows and columns with a zero right-hand side, as solve_body pins constant poses"""
    A, b = A.copy(), b.copy()
    A[idx, :] = 0.0
    A[:, idx] = 0.0
    A[idx, idx] = 1.0
    b[idx] = 0.0
    return A, b


def _make(kind, D, seed):
    rng = np.random.default_rng(seed)
    if kind.startswith("kappa"):
        A = _spd(rng, D, float(kind[5:]))
    elif kind == "spread":                # pose rows against bias rows: a row / column scaling of 1e-2 ... 1e4
        s = 10.0 ** rng.uniform(-2.0, 4.0, D)
        A = _spd(rng, D, 1e8) * np.outer(s, s)
    else:                                 # pinned unknowns at the start, in the middle and at the end
        A = _spd(rng, D, 1e4)
    b = A @ rng.standard_normal(D)
    if kind == "pinned":
        A, b = _pin(A, b, sorted({0, D // 2, D - 1}))
    return A, b


@functools.lru_cache(maxsize=None)
def _system(kind, D, seed):
    """(A, b, reference x, kappa_s) -- cached: every mode solves the same systems"""
    A, b = _make(kind, D, seed)
    return A, b, co.refined_solve(A, b), co.scaled_condition(A)


@functools.lru_cache(maxsize=None)
def _real_systems():
    """reduced systems of real windows, restricted to their free coordinates: the device's dump at mu = 0"""
    wins = {"cfg2": synth.make_cfg2()[:2], "cfg3": synth.make_cfg3()[:2],
            "cfg3_gauge": synth.make_cfg3(prior="gauge", N=6, M=120)[:2], "cfg4": synth.make_cfg4()[:2]}
    w, st, _ = synth.make_cfg3(N=6, M=100)
    st.bg = st.bg + np.array([2e-3, -1e-3, 1.5e-3])
    st.ba = st.ba + np.array([1e-2, 2e-2, -1e-2])
    wins["cfg3_bias"] = (w, st)
    b = BundleAdjustor(max_windows=1, max_frames=16, max_landmarks=640, max_obs=6000)
    out = {}
    for name, (w, st) in wins.items():
        o = b.gn_step(w, st, mu=0.0, want_system=True)
        free = bo.free_mask(w)[:15 * w.N]
        A, g = o["Hred"][np.ix_(free, free)], o["gred"][free]
        out[name] = (A, -g, co.refined_solve(A, -g), co.scaled_condition(A))
    b.close()
    return out


def _sweep(mode):
    """(label, nb, system) for every nb of the mode (D = 4 nb - 0 ... 3: every padding count) and kind, the production
    sizes of the mode and the real windows that fit it"""
    out = []
    for nb in range(1, NB_MAX[mode] + 1):
        for k, kind in enumerate(KINDS):
            D = max(1, 4 * nb - (nb + k) % 4)
            out.append((f"{kind} D={D}", nb, _system(kind, D, 1000 * D + k)))
    for i, D in enumerate(PROD_D[mode]):
        kind = KINDS[i % len(KINDS)]
        out.append((f"{kind} D={D} (production size)", (D + 3) // 4, _system(kind, D, 7 + D)))
    for name, s in _real_systems().items():
        if (len(s[1]) + 3) // 4 <= NB_MAX[mode]:
            out.append((name, (len(s[1]) + 3) // 4, s))
    return out


def _judge(label, A, b, x, xref, kappa):
    """backward error in units of D eps (asserted <= 4) and forward error over its bar (asserted <= 1)"""
    D = len(b)
    om = co.backward_error(A, x, b) / (D * EPS)
    fe = co.scaled_forward_error(x, xref, A) / (4 * D * EPS * max(kappa, 1.0))
    assert np.all(np.isfinite(x)) and om <= 4.0 and fe <= 1.0, (label, om, fe, kappa)
    return om, fe


@pytest.mark.parametrize("mode", sorted(NB_MAX))
def test_selftest_solves_every_block_count(ba, mode):
    cases = _sweep(mode)
    xs, ok = ba.selftest_chol([(A, b) for _, _, (A, b, _, _) in cases], mode)
    worst_om = worst_fe = 0.0
    for (label, nb, (A, b, xref, kappa)), x, k in zip(cases, xs, ok):
        assert k, (mode, label, nb)
        om, fe = _judge(f"{mode} nb={nb} {label}", A, b, x, xref, kappa)
        worst_om, worst_fe = max(worst_om, om), max(worst_fe, fe)
    nbs = sorted({nb for _, nb, _ in cases})
    assert nbs == list(range(1, NB_MAX[mode] + 1))
    print(f"chol {mode}: nb {nbs[0]} ... {nbs[-1]}, {len(cases)} systems; worst backward error {worst_om:.2f} D eps "
          f"(bar 4), worst forward error {worst_fe:.2e} of its bar")


def _bad_systems(rng):
    """systems whose factorisation must fail: a negative pivot in the first, a middle and the last block column, in the
    last real row of a padded tile, and a NaN entry"""
    out = []
    for D, k in ((40, 0), (40, 21), (40, 39), (38, 37)):
        A = _spd(rng, D, 1e4)
        A[k, k] = -1.0
        out.append((f"negative pivot at {k} of {D}", A, A @ rng.standard_normal(D)))
    A = _spd(rng, 40, 1e4)
    A[23, 9] = A[9, 23] = np.nan
    out.append(("NaN entry", A, rng.standard_normal(40)))
    return out


@pytest.mark.parametrize("mode", sorted(NB_MAX))
def test_failed_factorisation_is_reported_and_leaves_the_launch_alone(ba, mode):
    rng = np.random.default_rng(31)
    good = [_system(kind, D, 50 + D) for kind, D in (("kappa1e8", 13), ("spread", 40), ("pinned", 84))]
    bad = _bad_systems(rng)
    A17 = _spd(rng, 48, 1e17)                          # SPD, but its Schur complement may turn non-positive in rounding
    b17 = A17 @ rng.standard_normal(48)
    x_alone, ok_alone = ba.selftest_chol([s[:2] for s in good], mode)
    assert ok_alone.all()
    # launch order: bad 0, good 0, bad 1, bad 2, good 1, bad 3, good 2, bad 4, the kappa = 1e17 system
    tags = [("bad", 0), ("good", 0), ("bad", 1), ("bad", 2), ("good", 1), ("bad", 3), ("good", 2), ("bad", 4), ("k17", 0)]
    mixed = [good[i][:2] if t == "good" else bad[i][1:] if t == "bad" else (A17, b17) for t, i in tags]
    xs, ok = ba.selftest_chol(mixed, mode)
    for (t, i), x, k in zip(tags, xs, ok):
        if t == "good":
            assert k and np.array_equal(x, x_alone[i]), (mode, i)
        elif t == "bad":
            assert not k and np.all(x == 0.0), (mode, bad[i][0])
        elif k:                                        # either way, but ok and x agree
            _judge(f"{mode} kappa 1e17", A17, b17, x, x, 1.0)
        else:
            assert np.all(x == 0.0)
    print(f"chol {mode}: {len(bad)} non-SPD systems refused; kappa 1e17 system ok = {bool(ok[-1])}")


@pytest.mark.parametrize("mode", sorted(NB_MAX))
def test_selftest_is_deterministic_and_independent_of_its_neighbours(ba, mode):
    """the spin-wait publication of chol_solve_regs: a solve is bit-identical run twice, and at another position among
    other neighbours"""
    top = NB_MAX[mode]
    sizes = sorted({1, 5, 4 * min(top, 32), 4 * min(top, 33) - 1, 4 * top - 2, 4 * (top // 2) + 1, 6 * 8})
    systems = [_system(KINDS[i % len(KINDS)], D, 300 + D)[:2] for i, D in enumerate(sizes)]
    x1, ok1 = ba.selftest_chol(systems, mode)
    x2, ok2 = ba.selftest_chol(systems, mode)
    assert ok1.all() and ok2.all()
    assert all(np.array_equal(a, b) for a, b in zip(x1, x2))
    perm = np.random.default_rng(5).permutation(len(systems))
    extra = [_system("kappa1e12", D, 900 + D)[:2] for D in (4 * top - 1, 7, 4 * top)]
    batch = [extra[0]] + [systems[i] for i in perm[:3]] + [extra[1]] + [systems[i] for i in perm[3:]] + [extra[2]]
    x3, ok3 = ba.selftest_chol(batch, mode)
    assert ok3.all()
    pos = [1, 2, 3] + list(range(5, 5 + len(systems) - 3))
    for p, i in zip(pos, perm):
        assert np.array_equal(x3[p], x1[i]), (mode, len(systems[i][1]))


def test_selftest_rejects_what_production_does_not_run(ba):
    one = [(np.eye(4), np.ones(4))]
    with pytest.raises(PvioB200Error, match=EINVAL):
        ba.selftest_chol([(np.zeros((0, 0)), np.zeros(0))], "wide")
    for mode, D in (("narrow", 4 * 25), ("wide", 4 * 55), ("wide-tiled", 4 * 55)):
        ba.selftest_chol([(np.eye(D - 4), np.ones(D - 4))], mode)          # the largest block count still runs
        with pytest.raises(PvioB200Error, match=EINVAL):                   # one too large anywhere rejects the call
            ba.selftest_chol(one + [(np.eye(D), np.ones(D))], mode)
    D = np.array([4], dtype=np.int32)
    z = np.zeros(16)
    ok = np.zeros(1, dtype=np.int32)
    for n, mode in ((0, 1), (1, 3), (1, -1)):
        assert ba.lib.pvio_b200_selftest_chol(ba.h, n, mode, _lib.ptr(D), _lib.ptr(z), _lib.ptr(z), _lib.ptr(z),
                                              _lib.ptr(ok)) == _lib.EINVAL


def _production_check(ba, w, st, label, must_solve):
    """solve_kernel itself: at mu = 0 the regulariser is zero and the pinned rows are identity with g = 0, so dx over the
    free pose coordinates solves the dumped Hred[free, free] dx = -gred[free]"""
    P = 15 * w.N
    free = bo.free_mask(w)[:P]
    try:
        o = ba.gn_step(w, st, mu=0.0, want_system=True)
    except PvioB200Error as e:
        assert not must_solve and "not positive definite" in str(e), (label, str(e))
        return None
    A, b, x = o["Hred"][np.ix_(free, free)], -o["gred"][free], o["dx"][:P][free]
    om = co.backward_error(A, x, b) / (len(b) * EPS)
    assert om <= 4.0, (label, om)
    return om


def test_production_solve_meets_the_backward_error_bound(ba):
    """inertial N = 2 ... 11, single visual windows N = 2 ... 16 with 2, 1 and 0 fixed frames (with fewer than 2 the
    monocular gauge leaves the system singular: it may fail, and must meet the bar where it does not), a plane window and
    a gauge-prior window"""
    worst, n = 0.0, 0
    cases = [(f"inertial N={N}", synth.make_cfg3(N=N, M=60, seed=700 + N)[:2], True) for N in range(2, 12)]
    for N in range(2, 17):
        for nfix in (2, 1, 0):
            if N - nfix < 1:
                continue
            w, st, _ = synth.make_cfg2(N=N, M=60, seed=800 + N)
            w.frame_fixed[:] = 0
            w.frame_fixed[:nfix] = 1
            cases.append((f"visual N={N} fixed={nfix}", (w, st), nfix == 2))
    cases.append(("cfg4 planes", synth.make_cfg4()[:2], True))
    cases.append(("gauge prior", synth.make_cfg3(prior="gauge", N=6, M=120)[:2], True))
    for label, (w, st), must in cases:
        om = _production_check(ba, w, st, label, must)
        if om is not None:
            worst, n = max(worst, om), n + 1
    print(f"solve_kernel: {n} of {len(cases)} windows solved, worst backward error {worst:.2f} D eps (bar 4)")


def test_inertial_window_above_the_shared_memory_cap_is_refused_cleanly():
    """N = 11 needs 219,712 bytes of the 220 KB the solve kernel gets, N = 12 239,824: refused before any launch, and
    the same handle then solves an N = 11 window"""
    b = BundleAdjustor(max_windows=1, max_frames=12, max_landmarks=160, max_obs=2000)
    try:
        w12, s12, _ = synth.make_cfg3(N=12, M=80, seed=812)
        with pytest.raises(PvioB200Error, match=EINVAL):
            b.gn_step(w12, s12, mu=0.0)
        w, st, _ = synth.make_cfg3(N=11, M=80, seed=811)
        assert _production_check(b, w, st, "inertial N=11 after the refusal", True) is not None
    finally:
        b.close()
