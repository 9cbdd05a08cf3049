"""The hard-window generators of synthetic/synth.py and the oracle pieces they exercise, on the CPU: far and mixed
landmark depths, a tiny baseline, mismatched keypoints, a full 2x2 square-root information, Cauchy scales other than 1,
windows kilometres from the origin, landmarks the post-pass rejects and plane tracks off their plane.  Each generator
option is checked to produce what it claims, so the GPU tests built on them (test_gpu_ba_hard_windows.py) exercise the
kernel branches they are meant to; and the default generators are pinned bit for bit."""
import dataclasses
import hashlib

import numpy as np
import pytest

from oracle import ba_oracle as bo
from oracle import lie
from oracle import pnp_oracle as po
from synthetic import synth

EPS = 1e-6


def _fd(fun, x0_apply, n, eps=EPS):
    cols = []
    for i in range(n):
        d = np.zeros(n)
        d[i] = eps
        cols.append((fun(x0_apply(d)) - fun(x0_apply(-d))) / (2 * eps))
    return np.stack(cols, axis=-1)


def digest(obj, h=None):
    """sha256 over every array and scalar of a generator's output (dataclass fields and extra attributes, dict keys in
    sorted order), with dtypes and shapes."""
    top = h is None
    h = hashlib.sha256() if top else h
    if dataclasses.is_dataclass(obj):
        for f in dataclasses.fields(obj):
            h.update(f.name.encode())
            digest(getattr(obj, f.name), h)
        for k in sorted(set(vars(obj)) - {f.name for f in dataclasses.fields(obj)}):
            h.update(k.encode())
            digest(vars(obj)[k], h)
    elif isinstance(obj, dict):
        for k in sorted(obj):
            h.update(str(k).encode())
            digest(obj[k], h)
    elif isinstance(obj, (list, tuple)):
        h.update(b"[%d" % len(obj))
        for x in obj:
            digest(x, h)
    elif obj is None:
        h.update(b"None")
    else:
        a = np.ascontiguousarray(obj)
        h.update(str(a.dtype).encode() + str(a.shape).encode())
        h.update(a.tobytes())
    return h.hexdigest() if top else None


# taken before the hard-window options were added: the default windows, and so the golden files and every existing
# test, do not move
DEFAULT_DIGESTS = {
    "cfg2": "bf5f0b2f1d9a33cd9931938b355f9015ad61682959483e739aef841d3adc2890",
    "cfg3": "7fa822f0e2f9c1aa6566d348b20f6f57a72dae48545cfa3b9370057175945f16",
    "cfg4": "19d1726cb99b03abc966cc32789ecf3f267ee7d2396cdce70ffd80c51a451245",
    "pnp": "a795add459a543712c8d3f53a106c5dfe503f8e157bf9b484ece27854ae50bac",
}


@pytest.mark.parametrize("name", sorted(DEFAULT_DIGESTS))
def test_default_generators_unchanged(name):
    make = dict(cfg2=synth.make_cfg2, cfg3=synth.make_cfg3, cfg4=synth.make_cfg4, pnp=synth.make_pnp)[name]
    assert digest(make()) == DEFAULT_DIGESTS[name]


def test_general_sqrt_info_is_a_full_nonsymmetric_factor():
    w, _, _ = synth.make_cfg2(N=3, M=4)
    W = synth.general_sqrt_info(w)
    assert W[0, 1] != 0.0 and W[1, 0] != 0.0 and abs(W[0, 1] - W[1, 0]) > 0.1 * np.abs(W).max()
    assert abs(W[0, 0] - W[1, 1]) > 0.1 * np.abs(W).max()
    # the information it stands for: the diagonal one's pixel sigma, correlated
    sig = w.K_fx / w.sqrt_inv_cov[0, 0]
    Sig = np.linalg.inv(W.T @ W)
    assert np.isclose(np.sqrt(Sig[0, 0]) * w.K_fx, sig, rtol=1e-12)
    assert np.isclose(Sig[0, 1] / np.sqrt(Sig[0, 0] * Sig[1, 1]), 0.55, rtol=1e-12)


def test_reprojection_fd_general_w():
    """The oracle's reprojection functor with the full W, against finite differences (an index slip in W @ dproj or
    W @ r would show here)."""
    w, st, _ = synth.with_general_w(*synth.make_cfg2(N=4, M=6, staggered=True))
    W = w.sqrt_inv_cov
    for l in range(w.M):
        a = int(w.lm_anchor[l])
        for k in range(int(w.lm_obs_begin[l]), int(w.lm_obs_begin[l + 1])):
            t = int(w.obs_frame[k])

            def f(x):
                qt, pt, qr, pr, rho = x
                return bo.reprojection_evaluate(qt, pt, qr, pr, rho, w.obs_z[k], w.lm_z_ref[l],
                                                w.cam_q_cs, w.cam_p_cs, W, jac=False)[0]

            def app(d):
                return (lie.quat_plus(st.q[t], d[0:3]), st.p[t] + d[3:6],
                        lie.quat_plus(st.q[a], d[6:9]), st.p[a] + d[9:12], st.rho[l] + d[12])

            out = bo.reprojection_evaluate(st.q[t], st.p[t], st.q[a], st.p[a], st.rho[l], w.obs_z[k], w.lm_z_ref[l],
                                           w.cam_q_cs, w.cam_p_cs, W)
            J = np.hstack([out[1], out[2], out[3], out[4], out[5].reshape(2, 1)])
            assert np.allclose(J, _fd(f, app, 13), rtol=1e-5, atol=1e-4 * np.abs(J).max()), (l, k)
            # r = W (pi(y) - z): the transposed W gives another residual
            rT = bo.reprojection_evaluate(st.q[t], st.p[t], st.q[a], st.p[a], st.rho[l], w.obs_z[k], w.lm_z_ref[l],
                                          w.cam_q_cs, w.cam_p_cs, W.T, jac=False)[0]
            assert np.linalg.norm(rT - out[0]) > 1e-3 * np.linalg.norm(out[0])


@pytest.mark.parametrize("a", [1.0, 0.3, 0.01])
def test_corrector_gradient_fd(a):
    """The loss-corrected block (sqrt(rho') r, sqrt(rho') J) has the gradient of its cost rho(s)/2 = b/2 log(1 + s/b),
    b = a^2, at small residuals, at s ~ 1e6 and past t = 1 + s/b > 1e9 -- checked by finite differences of the cost."""
    w, _, st = synth.with_general_w(*synth.make_cfg2(N=3, M=4))      # at the truth: residuals of the pixel noise
    l, k = 1, int(w.lm_obs_begin[1])
    t, anc = int(w.obs_frame[k]), int(w.lm_anchor[l])
    seen = []
    for shift_px in (0.0, 30.0, 1500.0):
        z = w.obs_z[k] + np.array([shift_px / w.K_fx, 0.0])

        def cost(x):
            qt, pt = x
            r = bo.reprojection_evaluate(qt, pt, st.q[anc], st.p[anc], st.rho[l], z, w.lm_z_ref[l],
                                         w.cam_q_cs, w.cam_p_cs, w.sqrt_inv_cov, jac=False)[0]
            return np.array([bo.corrector_scale(r, a)[1]])

        out = bo.reprojection_evaluate(st.q[t], st.p[t], st.q[anc], st.p[anc], st.rho[l], z, w.lm_z_ref[l],
                                       w.cam_q_cs, w.cam_p_cs, w.sqrt_inv_cov)
        r, J = out[0], np.hstack([out[1], out[2]])
        s = float(r @ r)
        sc, c = bo.corrector_scale(r, a)
        assert np.isclose(c, 0.5 * a * a * np.log1p(s / (a * a)), rtol=1e-12)
        assert np.isclose(sc, 1.0 / np.sqrt(1.0 + s / (a * a)), rtol=1e-12)
        g = (sc * J).T @ (sc * r)
        gfd = _fd(cost, lambda d: (lie.quat_plus(st.q[t], d[0:3]), st.p[t] + d[3:6]), 6, eps=1e-7)[0]
        assert np.allclose(g, gfd, rtol=1e-5, atol=1e-6 * np.abs(g).max()), (shift_px, g, gfd)
        seen.append(s)
    assert seen[0] < 10 and 1e5 < seen[2] and seen[1] > 100     # a small residual, s ~ 1e6, and between
    if a == 0.01:
        assert 1 + seen[2] / (a * a) > 1e9


def _t_blocks(w, st):
    """1 + s/b of every reprojection block at st (b = cauchy_a^2)."""
    out = []
    for l in range(w.M):
        a = int(w.lm_anchor[l])
        for k in range(int(w.lm_obs_begin[l]), int(w.lm_obs_begin[l + 1])):
            t = int(w.obs_frame[k])
            r = bo.reprojection_evaluate(st.q[t], st.p[t], st.q[a], st.p[a], st.rho[l], w.obs_z[k], w.lm_z_ref[l],
                                         w.cam_q_cs, w.cam_p_cs, w.sqrt_inv_cov, jac=False)[0]
            out.append(1.0 + float(r @ r) / (w.cauchy_a ** 2))
    return np.array(out)


def test_outliers_and_small_cauchy_scale():
    base = synth.make_cfg2(N=6, M=60, seed=3)
    w, st, truth, bad = synth.with_outliers(*base, seed=1)
    nobs = np.diff(w.lm_obs_begin)
    whole = [l for l in range(w.M) if nobs[l] >= 2 and bad[w.lm_obs_begin[l]:w.lm_obs_begin[l + 1]].all()]
    assert len(whole) >= 2
    assert 0.05 * w.K <= bad.sum() <= 0.10 * w.K + nobs.max() * 2
    px = np.linalg.norm((w.obs_z - base[0].obs_z) * np.array([w.K_fx, w.K_fy]), axis=1)
    assert np.all(px[~bad] == 0) and px[bad].min() >= 15 - 1e-9 and px[bad].max() <= 300 + 1e-9
    assert np.array_equal(base[0].obs_z, synth.make_cfg2(N=6, M=60, seed=3)[0].obs_z)     # the input is not modified
    w01 = synth.with_cauchy(w, st, truth, 0.01)[0]
    t = _t_blocks(w01, st)
    assert np.sum(t > 1e9) >= 1 and np.sum(t <= 1e9) > 0.5 * len(t)          # both arms of LogAcc<float>::add
    assert bo.total_cost(w01, st) < bo.total_cost(w, st)


def test_rejected_landmarks_and_reprojection_error():
    w, st, truth, behind, far = synth.with_rejected_landmarks(*synth.make_cfg2(N=6, M=60, seed=4), seed=2)
    valid, quality = bo.landmark_postpass(w, st)
    assert not valid[behind].any() and not valid[far].any() and valid.sum() == w.M - 6
    assert np.all(st.rho[behind] < 0) and np.all(1.0 / truth.rho[far] > 50)
    # the far landmarks' observations agree with their new depth: at the truth the window costs what it did before
    w0, st0, t0 = synth.make_cfg2(N=6, M=60, seed=4)
    assert np.isclose(bo.total_cost(w, truth), bo.total_cost(w0, t0), rtol=0.05)
    # compute_reprojection_error counts every packed landmark; the mean of the post-pass qualities weighted by
    # observation count does not (a rejected landmark has quality 0 but is in the count)
    n = np.diff(w.lm_obs_begin) + 1
    e = bo.reprojection_error(w, st)
    assert abs(e - np.sum(quality * n) / np.sum(n)) > 1e-3 * e
    v0, q0 = bo.landmark_postpass(w0, st0)
    n0 = np.diff(w0.lm_obs_begin) + 1
    assert v0.all() and np.isclose(bo.reprojection_error(w0, st0), np.sum(q0 * n0) / np.sum(n0), rtol=1e-12)


def test_far_offset_is_a_pure_translation():
    for w, st, truth in (synth.make_cfg2(N=5, M=30, seed=5), synth.make_cfg3(N=5, M=40, seed=6),
                         synth.make_cfg4(N=5, M=30, seed=7, tracks_per_plane=20)):
        wo, so, to = synth.with_offset(w, st, truth)
        assert np.abs(so.p).max() > 1e3 and np.abs(to.p).max() > 1e3
        assert np.allclose(np.linalg.norm(so.p - st.p, axis=1), 5000.0, rtol=1e-3)
        # every reprojection, IMU and prior block costs what it did.  The plane blocks do not: the reference's
        # augmented plane functor regularises the triangulated point towards n.x = -d but measures n.x - d
        # (augmented_plane_distance_error_cost.h:84-96), so it is not translation invariant
        plane_moved = 0
        for (r, _, c), (ro, _, co) in zip(bo.iter_residual_blocks(w, st, jac=False),
                                         bo.iter_residual_blocks(wo, so, jac=False)):
            if len(r) == 1:
                plane_moved += abs(co - c) > 1e-6 * c
            else:
                assert abs(co - c) <= 1e-9 * max(c, 1e-9), (len(r), c, co)
        assert plane_moved == 0 if w.n_ptracks == 0 else plane_moved > 0
        if w.n_ptracks == 0:
            g, go = bo.gn_step(w, st)['dx'], bo.gn_step(wo, so)['dx']
            assert np.linalg.norm(go - g) <= 1e-6 * np.linalg.norm(g)


def test_depth_mixture_and_baseline():
    w, st, truth = synth.make_cfg2(N=6, M=100, seed=8, depth_mix=synth.DEPTH_MIX_OUTDOOR)
    d = 1.0 / truth.rho
    assert np.all((d[:70] >= 2) & (d[:70] <= 10))
    assert np.all((d[70:90] >= 20) & (d[70:90] <= 60))
    assert np.all((d[90:] >= 60) & (d[90:] <= 400)) and d.max() > 150
    valid, _ = bo.landmark_postpass(w, truth)
    assert not valid[90:].any() and valid[:70].all()
    w3, _, t3 = synth.make_cfg3(N=6, M=60, seed=9, depth_mix=((0.5, 20.0, 60.0), (0.5, 0.6, 1.0)))
    d3 = 1.0 / t3.rho
    assert np.all((d3[:30] >= 20) & (d3[:30] <= 60)) and np.all((d3[30:] >= 0.6) & (d3[30:] <= 1.0))
    ws, _, ts = synth.make_cfg2(N=6, M=20, seed=8, baseline=1e-3)
    _, _, tb = synth.make_cfg2(N=6, M=20, seed=8)
    assert np.allclose(ts.p, 1e-3 * tb.p, rtol=0, atol=1e-15) and np.linalg.norm(ts.p[-1] - ts.p[0]) < 2e-3


def test_offplane_tracks():
    base = synth.make_cfg4(N=6, M=30, seed=10, tracks_per_plane=20)
    w, st, truth, tracks, shift = synth.with_offplane_tracks(*base, seed=3)
    assert len(tracks) >= 10 and np.all((np.abs(shift) >= 0.3) & (np.abs(shift) <= 1.0))
    w0 = base[0]
    assert np.array_equal(w.pt_obs_frame, w0.pt_obs_frame)

    def tri(wz, t_):
        """the point the track's observations see from the truth poses (least-squares ray intersection)"""
        A, b = np.zeros((3, 3)), np.zeros(3)
        for k in range(int(w.pt_obs_begin[t_]), int(w.pt_obs_begin[t_ + 1])):
            f = int(w.pt_obs_frame[k])
            qc = lie.qmul(truth.q[f], w.cam_q_cs)
            pc = truth.p[f] + lie.qrot(truth.q[f], w.cam_p_cs)
            u = lie.qrot(qc, np.array([wz[k][0], wz[k][1], 1.0]))
            P = np.eye(3) - np.outer(u, u) / (u @ u)
            A += P
            b += P @ pc
        return np.linalg.solve(A, b)

    moved = 0
    for t_ in range(w.n_ptracks):
        n = w.plane_normal[w.pt_plane[t_]]
        dn = n @ (tri(w.pt_obs_z, t_) - tri(w0.pt_obs_z, t_))
        if t_ in tracks:
            s = shift[list(tracks).index(t_)]
            assert abs(dn - s) < 0.1 * abs(s), (t_, dn)     # the kept pixel noise, mapped through a short baseline
            moved += 1
        else:
            assert np.array_equal(w.pt_obs_z[w.pt_obs_begin[t_]:w.pt_obs_begin[t_ + 1]],
                                  w0.pt_obs_z[w0.pt_obs_begin[t_]:w0.pt_obs_begin[t_ + 1]])
    assert moved == len(tracks)
    # at those displacements the plane blocks' loss is far from quadratic (s = (100 x 0.3)^2 and more)
    assert (w.plane_sqrt_inv_cov * np.abs(shift).min()) ** 2 > 100


def test_pnp_options():
    d0 = synth.make_pnp()
    d = synth.make_pnp(depth=(30.0, 300.0), outlier_frac=0.08, W=synth.general_sqrt_info(synth._base_window(synth.EUROC, 2, True)),
                       cauchy_a=0.1, offset=synth.FAR_OFFSET)
    assert 'cauchy_a' not in d0 and d['cauchy_a'] == 0.1
    assert d['W'][0, 1] != 0 and d['W'][1, 0] != 0 and d['W'][0, 1] != d['W'][1, 0]
    assert np.abs(d['pts']).max() > 1e3 and np.abs(d['frame'][4:7]).max() > 1e3
    # the last frame sees the points at 30 - 300 m
    qc = lie.qmul(d['last'][0:4], d['cam_q'])
    pc = d['last'][4:7] + lie.qrot(d['last'][0:4], d['cam_p'])
    depth = np.array([lie.qrot(lie.qconj(qc), x - pc)[2] for x in d['pts']])
    assert depth.min() > 29 and depth.max() < 301 and depth.max() > 150
    z_clean = synth.make_pnp(depth=(30.0, 300.0))['zs']
    moved = np.linalg.norm((d['zs'] - z_clean) * np.array([synth.EUROC['K'][0], synth.EUROC['K'][1]]), axis=1)
    assert np.sum(moved > 0) == 12 and moved[moved > 0].min() >= 15 - 1e-9
    # pnp_solve passes cauchy_a to its problem: the costs differ as the loss says
    args = (d['last'], d['imu'], d['pts'], d['zs'], d['cam_q'], d['cam_p'], d['imu_q'], d['imu_p'], d['W'], True)
    c1 = po.PnpProblem(*args).cost(d['frame'])
    c01 = po.PnpProblem(*args, cauchy_a=0.1).cost(d['frame'])
    assert c01 < c1
    _, s1 = po.pnp_solve(d['frame'], *args, max_iter=1)
    _, s01 = po.pnp_solve(d['frame'], *args, max_iter=1, cauchy_a=0.1)
    assert s1['initial_cost'] == c1 and s01['initial_cost'] == c01


def test_hard_windows_of_the_gpu_tests_exercise_their_branches():
    """Preconditions of the exact windows test_gpu_ba_hard_windows.py builds (synth.hard_window, its default size)."""
    w, st = synth.hard_window("general_w")
    W = w.sqrt_inv_cov
    assert W[0, 1] != 0 and W[1, 0] != 0 and W[0, 1] != W[1, 0]           # the !diag_w branches
    w, st = synth.hard_window("cauchy_0.01")
    t = _t_blocks(w, st)
    assert t.max() > 1e9 and np.sum(t <= 1e9) > 0                          # both arms of LogAcc<float>::add
    w, st = synth.hard_window("offset")
    assert np.abs(st.p).max() > 1e3                                         # the origin shift matters
    w, st = synth.hard_window("rejected")
    assert np.sum(~bo.landmark_postpass(w, st)[0]) >= 6                     # the post-pass rejection branch
    w, st = synth.hard_window("far_depths")
    d = 1.0 / st.rho
    assert d.max() > 150 and np.sum(d > 20) >= 50
    w, st = synth.hard_window("low_baseline")
    assert np.linalg.norm(st.p[-1] - st.p[0]) < 0.05 and np.all(1.0 / st.rho > 1.5)     # 2 mm of travel + 1 cm guess noise
    for kind in synth.HARD_KINDS_INERTIAL:                                  # the inertial variants build too
        w, st = synth.hard_window(kind, inertial=True, N=8, M=200, seed=810)
        assert w.use_inertial and w.n_imu == 7
