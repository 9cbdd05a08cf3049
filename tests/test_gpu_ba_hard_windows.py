"""The bundle-adjustment, marginaliser and PnP kernels against the fp64 oracle on hard windows (synthetic/synth.py's
post-transforms, pinned on the CPU by test_hard_windows_oracle.py): landmarks at 20-400 m, a 1/1000 baseline,
mismatched keypoints, a full non-symmetric 2x2 square-root information, Cauchy scales 0.3 and 0.01 (t = 1 + s/b past
1e9), windows 5 km from the origin, landmarks the post-pass rejects and plane tracks off their plane -- each alone and
all at once, on a handle with fp32 records (visual only) and one with fp64 records (it has packed an inertial window).
The bars are the existing ones (test_gpu_ba.py, test_gpu_batch_marginalize.py, test_gpu_batch_pnp.py)."""
import numpy as np
import pytest

from oracle import ba_oracle as bo
from oracle import pnp_oracle as po
from synthetic import synth
from pvio_b200 import pnp
from pvio_b200.bundle_adjustor import BundleAdjustor

pytestmark = pytest.mark.gpu

TOL_DX = 1.0e-5
TERM = {'CONVERGENCE': 0, 'NO_CONVERGENCE': 1, 'FAILURE': 2}


def _rel(a, b):
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)


_f32_keypoints = synth.f32_keypoints
_base = synth.hard_base
make = synth.hard_window
VIS_KINDS, INE_KINDS = synth.HARD_KINDS_VISUAL, synth.HARD_KINDS_INERTIAL


@pytest.fixture(scope="module")
def ba32():
    """Visual-only windows only: the per-observation records stay fp32."""
    b = BundleAdjustor(max_windows=8, max_frames=10, max_landmarks=320, max_obs=3000)
    yield b
    b.close()


@pytest.fixture(scope="module")
def ba64():
    """Has packed an inertial window: fp64 records for good, for visual windows too."""
    b = BundleAdjustor(max_windows=8, max_frames=10, max_landmarks=320, max_obs=3000)
    w, st, _ = synth.make_cfg3(N=5, M=40, seed=1)
    b.gn_step(w, st)
    yield b
    b.close()


def _normal_equations_fp32_jacobians(win, st):
    """bo.normal_equations with every Jacobian block rounded to fp32: the precision floor the kernels' design accepts."""
    n = bo.local_dim(win)
    H, g, cost = np.zeros((n, n)), np.zeros(n), 0.0
    for r, blocks, c in bo.iter_residual_blocks(win, st):
        cost += c
        blocks = [(c0, J.astype(np.float32).astype(np.float64)) for c0, J in blocks]
        for ci, Ji in blocks:
            g[ci:ci + Ji.shape[1]] += Ji.T @ r
            for cj, Jj in blocks:
                H[ci:ci + Ji.shape[1], cj:cj + Jj.shape[1]] += Ji.T @ Jj
    return H, g, cost


def fp32_jacobian_yardstick(w, st, ref):
    """|dx(oracle, fp32 Jacobians) - dx(oracle)| / |dx(oracle)|, with the oracle's Jacobi scaling."""
    orig = bo.normal_equations
    bo.normal_equations = _normal_equations_fp32_jacobians
    try:
        y = bo.gn_step(w, st, scale=ref['scale'], schur=True)
    finally:
        bo.normal_equations = orig
    return _rel(y['dx'], ref['dx'])


def _check_step(ba, w, st, label, tol=TOL_DX, yardstick=True):
    """The bars of test_gpu_ba.py::_check_step; prints the worst errors and the fp32-Jacobian yardstick."""
    ref = bo.gn_step(w, st, schur=True)
    out = ba.gn_step(w, st, mu=1e-8, want_system=True)
    P = 15 * w.N
    e_pose, e_lm, e_all = _rel(out['dx'][:P], ref['dx'][:P]), _rel(out['dx'][P:], ref['dx'][P:]), _rel(out['dx'], ref['dx'])
    e_cost = abs(out['cost'] - ref['cost']) / ref['cost']
    cand = bo.total_cost(w, bo.apply_step(w, st, ref['dx']))
    e_cand = abs(out['new_cost'] - cand) / max(cand, 1.0)
    free = ref['free'][:P]
    Href = bo.gn_step(w, st, mu=0.0, schur=True)
    hs = np.sqrt(np.abs(np.diag(Href['Hred'])))[free]
    e_H = np.max(np.abs(out['Hred'][np.ix_(free, free)] - Href['Hred'][np.ix_(free, free)]) / np.outer(hs, hs))
    ys = fp32_jacobian_yardstick(w, st, ref) if yardstick else float('nan')
    print(f"{label}: N={w.N} M={w.M} K={w.K} dx pose {e_pose:.2e} lm {e_lm:.2e} all {e_all:.2e} | cost {e_cost:.2e} "
          f"cand {e_cand:.2e} Hred {e_H:.2e} | fp32-J yardstick {ys:.2e}")
    assert e_pose < tol and e_lm < tol and e_all < tol
    assert e_cost <= 2e-6
    assert np.all(out['dx'][~ref['free']] == 0.0)
    assert e_cand <= 5e-5
    assert e_H < 2e-5
    return out, ref


# ------------------------------------------------------------------ 1. gn_step, latency path
# The 1/1000-baseline window failed here before d r / d rho was formed as ir W dpi bt (ba_linearize.cuh): with fp32
# records the step was off by 1.2e-4 (fp32 Jacobians alone: 6e-8; cond(Jacobi-scaled Hred) = 7.7e2), the inverse-depth
# Jacobian G . (d x / d rho) cancelling to baseline / depth of its terms.
@pytest.mark.parametrize("kind", VIS_KINDS)
@pytest.mark.parametrize("records", ["fp32", "fp64"])
def test_gn_step_visual(ba32, ba64, kind, records):
    w, st = make(kind)
    _check_step(ba32 if records == "fp32" else ba64, w, st, f"{kind} visual {records}")


@pytest.mark.parametrize("kind", INE_KINDS)
def test_gn_step_inertial(ba64, kind):
    w, st = make(kind, inertial=True, N=8, M=200, seed=810)
    _check_step(ba64, w, st, f"{kind} inertial")


# ------------------------------------------------------------------ 2. throughput path
def _throughput(kinds, W, Nmax, Mmax, Kmax):
    b = BundleAdjustor(max_windows=W, max_frames=Nmax, max_landmarks=Mmax, max_obs=Kmax)
    try:
        for i in range(W):
            b.batch_set(i, *kinds[i % len(kinds)][1])
        b.batch_upload(W)
        b.batch_gn_step(W, 1e-8, apply=False)
        dx, costs = b.batch_download(W, 15 * Nmax + Mmax)
    finally:
        b.close()
    return dx, costs


@pytest.mark.parametrize("inertial", [False, True])
def test_throughput_heterogeneous_hard_batch(inertial):
    """88 windows, one CTA each, hard kinds interleaved with a normal one; visual only (fp32 records, lean solve
    kernel) or with inertial kinds (fp64 records).  Every kind's first and last window against its oracle step, and
    replicas against each other."""
    kinds = [(k, make(k, N=7, M=120, seed=820 + i)) for i, k in
             enumerate(["plain", "outliers", "general_w", "cauchy_0.01", "offset", "rejected", "far_depths", "all"])]
    if inertial:
        kinds += [(k + "_ine", make(k, inertial=True, N=7, M=120, seed=840 + i)) for i, k in
                  enumerate(["outliers", "offset", "all"])]
    W = 88
    dx, costs = _throughput(kinds, W, 8, 128, 1200)
    for k, (name, (w, st)) in enumerate(kinds):
        ref = bo.gn_step(w, st, schur=True)
        n = 15 * w.N + w.M
        first, last = k, k + len(kinds) * ((W - 1 - k) // len(kinds))
        errs = []
        for i in (first, last):
            errs.append(_rel(dx[i, :n], ref['dx']))
            assert errs[-1] < TOL_DX, (name, i, errs[-1])
            assert abs(costs[i, 0] - ref['cost']) <= 2e-6 * ref['cost'], (name, i)
        if inertial:
            assert np.allclose(dx[first], dx[last], rtol=1e-10, atol=0), name
        else:
            assert np.array_equal(dx[first], dx[last]) and np.array_equal(costs[first], costs[last]), name
        print(f"batch {'inertial' if inertial else 'visual'} {name}: dx rel err {max(errs):.2e}")


# ------------------------------------------------------------------ 3. trust-region solve
SOLVE_KINDS = ["outliers", "general_w", "far_depths", "offset", "all"]


def _check_solve(out, summ, ref_state, ref_sum, st, label, cost_tol=1e-5, state_tol=1e-5):
    e_cost = abs(summ['final_cost'] - ref_sum['final_cost']) / ref_sum['final_cost']
    move = max(np.linalg.norm(ref_state.p - st.p), 1e-3)
    e_p = np.linalg.norm(out.p - ref_state.p) / move
    e_rho = np.linalg.norm(out.rho - ref_state.rho) / max(np.linalg.norm(ref_state.rho - st.rho), 1e-300)
    print(f"{label}: iterations {summ['iterations']} / {ref_sum['iterations']}, accepted {summ['accepted_steps']} / "
          f"{sum(ref_sum['accepted'])}, final cost {e_cost:.2e}, state p {e_p:.2e} rho {e_rho:.2e}")
    assert summ['iterations'] == ref_sum['iterations']
    assert summ['accepted_steps'] == sum(ref_sum['accepted'])
    assert summ['termination'] == TERM[ref_sum['termination']]
    assert e_cost <= cost_tol
    assert e_p < state_tol + 1e-9 / move
    assert np.linalg.norm(out.rho - ref_state.rho) < state_tol * np.linalg.norm(ref_state.rho - st.rho) + 1e-9


def _solve_cases():
    cases = [(k, make(k, N=6, M=100, seed=860 + i)) for i, k in enumerate(SOLVE_KINDS)]
    cases.append(("offset_inertial", make("offset", inertial=True, N=6, M=100, seed=870)))
    return cases


def _batch_solve(refs):
    """batch_solve of the windows of refs on a handle of their own, each against its oracle solve"""
    b = BundleAdjustor(max_windows=len(refs), max_frames=6, max_landmarks=100, max_obs=600)
    try:
        for i, (_, w, st, _, _) in enumerate(refs):
            b.batch_set(i, w, st)
        b.batch_upload(len(refs))
        b.batch_solve(len(refs), max_iterations=6)
        frames, rho, sm = b.batch_download_state(len(refs), 6, 100)
    finally:
        b.close()
    for i, (name, w, st, ref_state, ref_sum) in enumerate(refs):
        out = st.copy()
        out.q, out.p, out.v, out.bg, out.ba = (frames[i, :, a:b] for a, b in ((0, 4), (4, 7), (7, 10), (10, 13), (13, 16)))
        out.rho = rho[i, :w.M]
        _check_solve(out, sm[i], ref_state, ref_sum, st, f"batch_solve {name}")


def test_solve_matches_oracle(ba32, ba64):
    """ba.solve on each kind (visual kinds with fp32 records), then the device-side loop over a batch of the visual
    kinds with fp32 records and over all kinds with fp64 records (the inertial window switches that handle)."""
    refs = []
    for name, (w, st) in _solve_cases():
        ref_state, ref_sum = bo.solve(w, st, max_iter=6)
        refs.append((name, w, st, ref_state, ref_sum))
        out, summ = (ba64 if w.use_inertial else ba32).solve(w, st, max_iterations=6, postpass=False)
        _check_solve(out, summ, ref_state, ref_sum, st, name)
    _batch_solve([r for r in refs if not r[1].use_inertial])
    _batch_solve(refs)


def test_solve_dogleg_small_radius_outliers_general_w(ba32):
    """The Gauss-Newton step leaves a radius-2 region: the Cauchy point's J.v sweep (jv_vision_kernel) runs with the full
    W and the outliers' loss scaling.  The bars of test_solve_dogleg_and_rejections_match_oracle."""
    base = _base(False, "outliers", 6, 80, 880)
    w, st, truth, _ = synth.with_outliers(*base, seed=6)
    w, st, truth = synth.with_general_w(w, st, truth)
    w = _f32_keypoints(w)
    r0 = 2.0
    # precondition: the first Gauss-Newton step, in the Jacobi-scaled coordinates the trust region measures
    # (bo.trust_region: |gn_s| with dx = gn_s / diag * scale), is longer than the radius: the dogleg leg runs
    g0 = bo.gn_step(w, st)
    idx = np.where(g0['free'])[0]
    sc = g0['scale'][idx]
    diag = np.sqrt(np.clip(sc * sc * np.diag(g0['H'])[idx], bo.MIN_DIAG, bo.MAX_DIAG))
    gn_norm = np.linalg.norm(g0['dx'][idx] * diag / sc)
    print(f"dogleg: scaled Gauss-Newton step {gn_norm:.3e} against radius {r0}")
    assert gn_norm > 2.0 * r0
    ref_state, ref_sum = bo.solve(w, st, max_iter=8, radius0=r0)
    out, summ = ba32.solve(w, st, max_iterations=8, initial_radius=r0, postpass=False)
    _check_solve(out, summ, ref_state, ref_sum, st, "dogleg r0=2", cost_tol=5e-5, state_tol=2e-5)


# ------------------------------------------------------------------ 4. post-pass and reprojection error
@pytest.mark.parametrize("inertial", [False, True])
def test_postpass_and_reprojection_error(ba64, inertial):
    base = _base(inertial, "rejected", 6, 100, 890)
    w, st, truth, behind, far = synth.with_rejected_landmarks(*base, seed=7)
    w, st, truth, _ = synth.with_outliers(w, st, truth, seed=8)
    w, st, truth = synth.with_offset(w, st, truth)
    w = _f32_keypoints(w)
    assert np.sum(~bo.landmark_postpass(w, st)[0]) >= len(behind) + len(far)
    out, summ = ba64.solve(w, st, max_iterations=3)
    valid, quality = bo.landmark_postpass(w, out)          # the oracle's post-pass at the kernel's own final state
    assert np.sum(~valid) >= 3                              # the rejection branch still runs at the solution
    assert np.array_equal(summ['valid'], valid)
    e_q = np.max(np.abs(summ['quality'][valid] - quality[valid]) / quality[valid])
    assert np.all(summ['quality'][~valid] == 0.0)
    e = ba64.compute_reprojection_error(w, st)
    ref = bo.reprojection_error(w, st)
    print(f"post-pass: {np.sum(~valid)} of {w.M} rejected, quality rel err {e_q:.2e}, reprojection error "
          f"{abs(e - ref) / ref:.2e}")
    assert e_q < 1e-6
    assert abs(e - ref) <= 1e-9 * ref


# ------------------------------------------------------------------ 5. marginaliser
NOISE_ABS = 1.0e-7          # see test_gpu_batch_marginalize.py


def _check_prior(S, e, S1, e1, H1, tol):
    hs = np.maximum(np.sqrt(np.abs(np.diag(H1))), 1e-3)
    L, L1 = S.T @ S, S1.T @ S1
    eL = np.max(np.abs(L - L1) / (tol * np.outer(hs, hs) + NOISE_ABS))
    ev = np.max(np.abs(S.T @ e - S1.T @ e1)) / np.max(np.abs(S1.T @ e1))
    ev_ = np.linalg.eigvalsh(0.5 * (H1 + H1.T))
    n_noise = int(np.sum((np.abs(ev_) > 1e-10) & (np.abs(ev_) < 1e-6)))
    n_pos = lambda X: int(np.sum(np.linalg.norm(X, axis=1) > 0))
    assert eL < 1.0 and ev < tol, (eL, ev)
    assert abs(n_pos(S) - n_pos(S1)) <= n_noise
    return eL, ev


def test_marginalize_hard_windows():
    kinds = [(k, make(k, inertial=True, N=6, M=150, seed=900 + i)) for i, k in
             enumerate(["outliers", "far_depths", "offset", "all"])]
    b = BundleAdjustor(max_windows=len(kinds), max_frames=6, max_landmarks=160, max_obs=1200)
    try:
        singles = [b.marginalize_frame(w, st, 0, want_info=True) for _, (w, st) in kinds]
        for i, (_, (w, st)) in enumerate(kinds):
            b.batch_set(i, w, st)
        b.batch_upload(len(kinds))
        batch = b.batch_marginalize(len(kinds), want=True)
    finally:
        b.close()
    for (name, (w, st)), (S, e, H, bv), (Sb, eb) in zip(kinds, singles, batch):
        S0, e0, H0, b0 = bo.marginalize(w, st, index=0)
        hs = np.maximum(np.sqrt(np.abs(np.diag(H0))), 1e-3)
        eH = np.max(np.abs(H - H0) / np.outer(hs, hs))
        eb_ = np.max(np.abs(bv - b0)) / np.max(np.abs(b0))
        eL, ev = _check_prior(S, e, S0, e0, H0, 1e-6)
        eLb, evb = _check_prior(Sb, eb, S, e, H, 1e-9)
        print(f"marginalise {name}: H {eH:.2e} b {eb_:.2e} S^T S {eL:.2e} (of the bar) S^T e {ev:.2e}; "
              f"batch vs single {eLb:.2e} {evb:.2e}")
        assert eH < 1e-6 and eb_ < 1e-6


# ------------------------------------------------------------------ 6. planes
def _planes(seed):
    base = synth.make_cfg4(N=6, M=60, seed=seed, tracks_per_plane=20)
    w, st, truth, _, _ = synth.with_offplane_tracks(*base, seed=9)
    w, st, truth = synth.with_offset(w, st, truth)
    return _f32_keypoints(w), st


def test_planes_offplane_and_offset(ba64):
    w, st = _planes(910)
    _check_step(ba64, w, st, "cfg4 off-plane + offset")
    ref_state, ref_sum = bo.solve(w, st, max_iter=6)
    out, summ = ba64.solve(w, st, max_iterations=6, postpass=False)
    _check_solve(out, summ, ref_state, ref_sum, st, "cfg4 off-plane + offset solve")


# ------------------------------------------------------------------ 7. PnP
def _pnp_cases():
    W = synth.general_sqrt_info(synth._base_window(synth.EUROC, 2, True))
    specs = [dict(outlier_frac=0.08), dict(W=W), dict(outlier_frac=0.08, W=W, cauchy_a=0.1),
             dict(depth=(30.0, 300.0)), dict(offset=synth.FAR_OFFSET),
             dict(depth=(30.0, 300.0), outlier_frac=0.08, W=W, cauchy_a=0.1, offset=synth.FAR_OFFSET)]
    out = []
    for i, kw in enumerate(specs):
        for inertial in (True, False):
            d = synth.make_pnp(seed=920 + 2 * i + inertial, use_inertial=inertial, **kw)
            d['zs'] = d['zs'].astype(np.float64)
            out.append((f"{sorted(kw)} inertial={inertial}", d))
    return out


def _pnp_oracle(d):
    return po.pnp_solve(d['frame'], d['last'], d['imu'], d['pts'], d['zs'], d['cam_q'], d['cam_p'], d['imu_q'],
                        d['imu_p'], d['W'], d['use_inertial'], cauchy_a=d.get('cauchy_a', 1.0))


def _check_pnp(name, d, xg, sg, xr, sr):
    e_cost = abs(sg['final_cost'] - sr['final_cost']) / sr['final_cost']
    move = max(np.linalg.norm(xr - d['frame']), 1e-3)
    e_x = np.linalg.norm(xg - xr) / move
    print(f"pnp {name}: iterations {sg['iterations']} / {sr['iterations']}, cost {e_cost:.2e}, state {e_x:.2e}")
    assert sg['iterations'] == sr['iterations'] and sg['accepted_steps'] == sum(sr['accepted'])
    assert abs(sg['initial_cost'] - sr['initial_cost']) <= 1e-9 * sr['initial_cost']
    assert e_cost <= 1e-9
    assert e_x < 1e-8


def test_pnp_hard_inputs(ba32):
    cases = _pnp_cases()
    refs = [_pnp_oracle(d) for _, d in cases]
    for (name, d), (xr, sr) in zip(cases, refs):
        xg, sg = pnp.visual_inertial_pnp(ba32, d['frame'], d['last'], d['imu'], d['pts'], d['zs'], d['cam_q'],
                                         d['cam_p'], d['imu_q'], d['imu_p'], d['W'], d['use_inertial'],
                                         cauchy_a=d.get('cauchy_a', 1.0))
        _check_pnp(name, d, xg, sg, xr, sr)
    xs, sums = pnp.batch_visual_inertial_pnp(ba32, [d for _, d in cases])
    for (name, d), (xr, sr), xg, sg in zip(cases, refs, xs, sums):
        _check_pnp("batch " + name, d, xg, sg, xr, sr)
