"""pvio_b200_batch_marginalize: BundleAdjustor::marginalize_frame(0) (bundle_adjustor.cpp:348-599) for a whole batch of
uploaded windows at their device states, each window's new prior kept in its own slot on the device.  Checked against the
single-window marginaliser, the oracle, the host-prior path, and a keyframe cycle of independent sequences."""
import dataclasses

import numpy as np
import pytest

from oracle import ba_oracle as bo
from synthetic import synth
from synthetic.sequence import Run, Chain
from pvio_b200 import _lib
from pvio_b200.bundle_adjustor import BundleAdjustor, PvioB200Error
from pvio_b200.window import State

pytestmark = pytest.mark.gpu

EINVAL = rf"error {_lib.EINVAL}\b"


def _rel(a, b):
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)


# A window whose information has a null space (here: after the 1e15 gauge prior's frame leaves, yaw and position are
# unobservable) has eigenvalues that are rounding noise, |lambda| ~ 4e-8 at lambda_max ~ 2e8, on both sides of the
# reference's 1e-8 clamp.  Two runs of the SAME single-window marginaliser, whose system differs in the last bits (fp64
# atomics of the linearise sweep), then keep different noise directions: measured on an H100, S^T S differed by up to
# 3e-8 absolute in coordinates without information, 3e-2 in the scaled metric of test_marginalize_matches_oracle (whose
# floor hs = 1e-3 makes hs^2 = 1e-6), and the count of positive directions by 1 (against the oracle by 3).  So S^T S is
# compared with an absolute allowance of 1e-7 beside the scaled bar, and the positive counts up to the number of noise
# eigenvalues.  Windows without such a null space are held to the scaled bar alone: their runs differ by 6e-12.
NOISE_ABS = 1.0e-7


def _info_err(S, e, S1, e1, hs, tol, noise_abs=NOISE_ABS):
    """(max |S^T S - S1^T S1| / (tol hs hs^T + noise_abs), relative max |S^T e - S1^T e1|).  S is unique only up to the
    sign / order of its rows."""
    L, L1 = S.T @ S, S1.T @ S1
    v, v1 = S.T @ e, S1.T @ e1
    return np.max(np.abs(L - L1) / (tol * np.outer(hs, hs) + noise_abs)), np.max(np.abs(v - v1)) / np.max(np.abs(v1))


def _n_pos(S):
    return int(np.sum(np.linalg.norm(S, axis=1) > 0))


def _n_noise(H):
    """eigenvalues of the marginalised system H that are rounding noise around the 1e-8 clamp"""
    ev = np.linalg.eigvalsh(0.5 * (H + H.T))
    return int(np.sum((np.abs(ev) > 1e-10) & (np.abs(ev) < 1e-6)))


def _check_prior(S, e, S1, e1, H1, tol, noise_abs=NOISE_ABS):
    hs = np.maximum(np.sqrt(np.abs(np.diag(H1))), 1e-3)
    eL, ev = _info_err(S, e, S1, e1, hs, tol, noise_abs)
    assert eL < 1.0 and ev < tol, (eL, ev)
    assert abs(_n_pos(S) - _n_pos(S1)) <= _n_noise(H1), (_n_pos(S), _n_pos(S1), _n_noise(H1))
    return eL, ev


def _with_marg_prior(w, st, S=None, e=None):
    """The window carrying the prior that marginalising its frame 0 at `st` leaves, over frames 1 .. N - 1 (the victim
    stays in the window, as in test_marginalize_then_solve_chain).  Without S / e the prior is the device-resident one:
    zeros keep Window.validate()'s shapes, batch_set(resident_prior=True) does not send them."""
    keep = np.arange(1, w.N)
    d = 15 * (w.N - 1)
    w2 = dataclasses.replace(w)
    w2.n_prior = w.N - 1
    w2.prior_frames = keep.astype(np.int32)
    w2.prior_S = np.zeros((d, d)) if S is None else S
    w2.prior_e = np.zeros(d) if e is None else e
    w2.prior_q0, w2.prior_p0, w2.prior_v0 = st.q[keep].copy(), st.p[keep].copy(), st.v[keep].copy()
    w2.prior_bg0, w2.prior_ba0 = st.bg[keep].copy(), st.ba[keep].copy()
    w2.validate()
    st2 = st.copy()
    st2.p[1:] += 1e-3
    return w2, st2


def _kinds8():
    """8 distinct inertial windows: N in {6, 9}, the 1e15 gauge prior, a full N - 1 prior, none."""
    return [synth.make_cfg3(N=9, seed=648)[:2], synth.make_cfg3(N=6, M=200, seed=649)[:2],
            synth.make_cfg3(N=9, seed=650, prior='gauge')[:2], synth.make_cfg3(N=6, M=200, seed=651, prior='gauge')[:2],
            synth.make_cfg3(N=9, M=250, seed=652)[:2], synth.make_cfg3(N=6, M=150, seed=653)[:2],
            synth.make_cfg3(N=9, M=300, seed=654, prior='none')[:2], synth.make_cfg3(N=6, M=200, seed=655)[:2]]


@pytest.fixture(scope="module")
def kinds():
    return _kinds8()


@pytest.fixture(scope="module")
def bat():
    b = BundleAdjustor(max_windows=8, max_frames=9, max_landmarks=320, max_obs=3000)
    yield b
    b.close()


def test_batch_marginalize_matches_single_window_and_oracle(bat, kinds):
    """Every window of a batch of 8 distinct windows gets the prior its own pvio_b200_ba_marginalize gives it; S_out / e_out
    are the priors the slots keep on the device."""
    singles = [bat.marginalize_frame(w, st, 0, want_info=True) for w, st in kinds]
    for i, (w, st) in enumerate(kinds):
        bat.batch_set(i, w, st)
    bat.batch_upload(8)
    out = bat.batch_marginalize(8, want=True)
    worst = [0.0, 0.0]
    for i, (w, st) in enumerate(kinds):
        S, e = out[i]
        S1, e1, H1, _ = singles[i]
        assert S.shape == (15 * (w.N - 1),) * 2 and e.shape == (15 * (w.N - 1),)
        eL, ev = _check_prior(S, e, S1, e1, H1, 1e-9)
        worst = [max(worst[0], eL), max(worst[1], ev)]
        # against the oracle: the bars of test_marginalize_matches_oracle
        S0, e0, H0, _ = bo.marginalize(w, st, index=0)
        _check_prior(S, e, S0, e0, H0, 1e-6)
    print("batch vs single-window marginaliser: worst S^T S %.2e (of the bar), S^T e %.2e" % tuple(worst))
    # the slot's device prior is S_out / e_out: a GN step of each window with the resident prior equals the same window
    # packed with S_out / e_out as a host prior
    stride = 15 * 9 + 320
    for i, (w, st) in enumerate(kinds):
        bat.batch_set(i, *_with_marg_prior(w, st), resident_prior=True)
    bat.batch_upload(8)
    bat.batch_gn_step(8, 1e-8)
    dx_res, c_res = bat.batch_download(8, stride)
    for i, (w, st) in enumerate(kinds):
        bat.batch_set(i, *_with_marg_prior(w, st, *out[i]))
    bat.batch_upload(8)
    bat.batch_gn_step(8, 1e-8)
    dx_host, c_host = bat.batch_download(8, stride)
    for i, (w, _) in enumerate(kinds):
        n = 15 * w.N + w.M
        assert _rel(dx_res[i, :n], dx_host[i, :n]) < 1e-9, i
        assert abs(c_res[i, 0] - c_host[i, 0]) <= 1e-9 * c_host[i, 0], i


def test_batch_marginalize_over_several_chunks():
    """300 windows are more than one pass of the dense kernels (2 per SM); each equals its kind's single-window prior."""
    W = 300
    b = BundleAdjustor(max_windows=W, max_frames=6, max_landmarks=160, max_obs=1200)
    kinds = [synth.make_cfg3(N=6, M=120, seed=660 + i, prior=p)[:2] for i, p in enumerate(('synthetic', 'gauge', 'none'))]
    singles = [b.marginalize_frame(w, st, 0, want_info=True) for w, st in kinds]
    for i in range(W):
        b.batch_set(i, *kinds[i % 3])
    b.batch_upload(W)
    out = b.batch_marginalize(W, want=True)
    for i in range(W):
        S1, e1, H1, _ = singles[i % 3]
        _check_prior(*out[i], S1, e1, H1, 1e-9)
    b.close()


class _ResidentChain(Chain):
    """Chain whose prior after the first keyframe is the one batch_marginalize left in the sequence's slot."""
    resident = False

    def keep_resident_prior(self, k):
        N = self.run.N
        d = 15 * (N - 1)
        self.prior = dict(frames=list(range(k + 1, k + N)), S=np.zeros((d, d)), e=np.zeros(d), x0=np.zeros((N - 1, 16)))
        self.resident = True


def test_batched_keyframe_cycle_follows_the_repacked_sequences():
    """4 independent sequences (N = 6, 6, 8, 8) through 10 keyframes of batch_set (shifted window, resident prior) ->
    batch_upload -> batch_solve -> batch_download_state -> batch_marginalize, against each sequence re-packed window by
    window through ba_solve + ba_marginalize with the prior carried through the host."""
    runs = [Run(F=18, N=6, M=220, seed=710), Run(F=18, N=6, M=220, seed=711),
            Run(F=20, N=8, M=260, seed=712), Run(F=20, N=8, M=260, seed=713)]
    bat = BundleAdjustor(max_windows=4, max_frames=8, max_landmarks=320, max_obs=3000)
    one = BundleAdjustor(max_windows=1, max_frames=8, max_landmarks=320, max_obs=3000)
    gpu, ref = [_ResidentChain(r) for r in runs], [Chain(r) for r in runs]
    worst = 0.0
    for k in range(10):
        views = []
        for j, c in enumerate(gpu):
            w, st, ids = c.window(k)
            bat.batch_set(j, w, st, resident_prior=c.resident)
            views.append((w, ids))
        bat.batch_upload(4)
        bat.batch_solve(4, max_iterations=6)
        frames, rho, sm = bat.batch_download_state(4, 8, 320)
        bat.batch_marginalize(4)
        for j, (w, ids) in enumerate(views):
            wr, sr, ids_r = ref[j].window(k)
            assert ids == ids_r, (k, j)
            out, summ = one.solve(wr, sr, max_iterations=6, postpass=False)
            S, e = one.marginalize_frame(wr, out, index=0)
            ref[j].store(k, out, ids_r)
            ref[j].set_prior(k, S, e, out)
            assert sm[j]['iterations'] == summ['iterations'] and sm[j]['accepted_steps'] == summ['accepted_steps'], (k, j)
            fr = frames[j, :w.N]
            st = State(fr[:, 0:4], fr[:, 4:7], fr[:, 7:10], fr[:, 10:13], fr[:, 13:16], rho[j, :w.M].copy())
            refv = np.concatenate([out.q, out.p, out.v, out.bg, out.ba], axis=1)
            worst = max(worst, np.abs(fr - refv).max(), np.max(np.abs(st.rho - out.rho) / np.abs(out.rho)))
            gpu[j].store(k, st, ids)
            gpu[j].keep_resident_prior(k)
    bat.close()
    one.close()
    print("batched keyframe cycle vs re-packed sequences: worst state / inverse-depth difference", worst)
    # Measured on an H100: the re-packed single-window chain run twice on two handles differs by up to 1.3e-7 in position
    # and 5.4e-7 in relative inverse depth after 10 keyframes (sequences 711 and 713; 4e-10 for 710 and 712): last-bit
    # differences of the fp64 atomics grow through the solves and through the priors' noise directions (NOISE_ABS above).
    # The batched cycle stayed inside that spread (1.3e-7, 1.9e-7); the bar is four times the spread.
    assert worst < 2e-6


def _unchanged(b, n, N, M):
    fr, rho, sm = b.batch_download_state(n, N, M)
    return fr.copy(), rho.copy(), [dict(x) for x in sm]


def _same(a, b):
    return np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and a[2] == b[2]


def test_rejected_calls_change_nothing(kinds):
    b = BundleAdjustor(max_windows=4, max_frames=13, max_landmarks=320, max_obs=3000)
    (w0, s0), (w1, s1) = kinds[0], kinds[1]
    wv, sv, _ = synth.make_cfg2(N=6, M=80, seed=661)
    for i, (w, st) in enumerate(((w0, s0), (w1, s1), (wv, sv))):
        b.batch_set(i, w, st)
    b.batch_upload(3)
    b.batch_solve(3, max_iterations=4)
    snap = _unchanged(b, 3, 9, 320)
    with pytest.raises(PvioB200Error, match=EINVAL):            # a visual-only window in the batch
        b.batch_marginalize(3)
    assert _same(_unchanged(b, 3, 9, 320), snap)
    with pytest.raises(PvioB200Error, match=EINVAL):            # the rejected call left no resident prior behind
        b.batch_set(0, *_with_marg_prior(w0, s0), resident_prior=True)
    assert _same(_unchanged(b, 3, 9, 320), snap)
    with pytest.raises(PvioB200Error, match=EINVAL):            # n > n_uploaded
        b.batch_marginalize(4)
    assert _same(_unchanged(b, 3, 9, 320), snap)
    S_all = b.batch_marginalize(2, want=True)                   # valid: the two inertial windows
    assert _same(_unchanged(b, 3, 9, 320), snap)                # the device states are not modified
    wbad, sbad = _with_marg_prior(w0, s0)                       # a different n_prior than the resident prior covers
    wbad = dataclasses.replace(wbad, n_prior=w0.N - 2, prior_frames=wbad.prior_frames[:-1],
                               prior_S=np.zeros((15 * (w0.N - 2),) * 2), prior_e=np.zeros(15 * (w0.N - 2)))
    with pytest.raises(PvioB200Error, match=EINVAL):
        b.batch_set(0, wbad, sbad, resident_prior=True)
    assert _same(_unchanged(b, 3, 9, 320), snap)
    with pytest.raises(PvioB200Error, match=EINVAL):            # slot 2 holds no resident prior
        b.batch_set(2, *_with_marg_prior(w1, s1), resident_prior=True)
    assert _same(_unchanged(b, 3, 9, 320), snap)
    b.batch_set(0, *_with_marg_prior(w0, s0), resident_prior=True)       # valid: names slot 0's resident prior
    with pytest.raises(PvioB200Error, match=EINVAL):            # slot 0's staging does not hold its prior
        b.batch_replicate(2)
    b.batch_set(1, *_with_marg_prior(w1, s1), resident_prior=True)
    b.batch_upload(2)                                           # the following valid calls succeed
    b.batch_gn_step(2, 1e-8)
    dx, _ = b.batch_download(2, 15 * 9 + 320)
    assert np.all(np.isfinite(dx))
    assert len(S_all) == 2
    # 13 frames (dk = 180) are more than the shared-memory eigen-solver takes: rejected alone and inside a batch
    w13, s13, _ = synth.make_cfg3(N=13, M=120, seed=662)
    b.batch_set(2, w13, s13)
    b.batch_upload(3)
    snap = _unchanged(b, 3, 13, 320)
    with pytest.raises(PvioB200Error, match=EINVAL):
        b.marginalize_frame(w13, s13, 0)
    assert _same(_unchanged(b, 3, 13, 320), snap)
    with pytest.raises(PvioB200Error, match=EINVAL):
        b.batch_marginalize(3)
    assert _same(_unchanged(b, 3, 13, 320), snap)
    b.close()


def test_slots_keep_their_resident_priors_independently(bat, kinds):
    """A slot re-packed with a host prior uploads that prior while its neighbours keep their device-resident ones."""
    ks = kinds[:3]
    for i, (w, st) in enumerate(ks):
        bat.batch_set(i, w, st)
    bat.batch_upload(3)
    pri = bat.batch_marginalize(3, want=True)
    # slot 1: a host prior unlike its resident one (the resident S scaled by 2)
    packs = [_with_marg_prior(*ks[0]), _with_marg_prior(*ks[1], 2.0 * pri[1][0], 2.0 * pri[1][1]), _with_marg_prior(*ks[2])]
    for i, (w, st) in enumerate(packs):
        bat.batch_set(i, w, st, resident_prior=(i != 1))
    bat.batch_upload(3)
    bat.batch_gn_step(3, 1e-8)
    stride = 15 * 9 + 320
    dx, _ = bat.batch_download(3, stride)
    ref = BundleAdjustor(max_windows=3, max_frames=9, max_landmarks=320, max_obs=3000)
    hosts = [_with_marg_prior(*ks[0], *pri[0]), packs[1], _with_marg_prior(*ks[2], *pri[2])]
    for i, (w, st) in enumerate(hosts):
        ref.batch_set(i, w, st)
    ref.batch_upload(3)
    ref.batch_gn_step(3, 1e-8)
    dx_ref, _ = ref.batch_download(3, stride)
    ref.close()
    for i, (w, _) in enumerate(ks):
        n = 15 * w.N + w.M
        assert _rel(dx[i, :n], dx_ref[i, :n]) < 1e-9, i
    # the scaled prior really changed slot 1's step
    w1, st1 = _with_marg_prior(*ks[1], *pri[1])
    assert _rel(bat.gn_step(w1, st1)['dx'], dx[1, :15 * w1.N + w1.M]) > 1e-6
