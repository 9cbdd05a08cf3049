"""oracle/trajectory_oracle.py, the reference of pvio_b200_batch_window_trajectory: at a factor's first sample the state
is the frame's own and the covariance the frame's; at t_end the increment is imu_oracle.integrate of the whole factor;
and the factor-selection rule at the gaps, at the boundaries and over factors without samples."""
import numpy as np

from oracle import imu_oracle
from oracle import imu_stream_cov_oracle as sco
from oracle import trajectory_oracle as to
from synthetic import synth


def _window(seed=880, N=6):
    w, st, truth = synth.make_cfg3(N=N, M=60, seed=seed)
    frames = np.concatenate([st.q, st.p, st.v, st.bg, st.ba], axis=1)
    factors = [(s.copy(), t) for s, t, _, _ in truth.imu_factors]
    rng = np.random.default_rng(seed)
    Sig = []
    for _ in range(N):
        A = rng.normal(size=(15, 15))
        Sig.append(A @ A.T * 1e-4)
    return frames, factors, truth.imu_noise, np.array(Sig)


def test_frame_time_gives_the_frame_state_and_covariance():
    frames, factors, noise, Sig = _window()
    t0 = [f[0][0, 0] for f in factors]
    fr, st, cov = to.trajectory(t0, frames, factors, noise, Sig)
    assert np.array_equal(fr, np.arange(len(factors)))
    for k in range(len(factors)):
        assert np.array_equal(st[k], frames[k]), k
        assert np.array_equal(cov[k], 0.5 * (Sig[k] + Sig[k].T)), k


def test_t_end_gives_the_full_factor():
    frames, factors, noise, Sig = _window()
    for k, (s, t_end) in enumerate(factors):
        x = frames[k]
        d = to.delta(s, t_end, x[10:13], x[13:16], noise)
        ref = imu_oracle.integrate(s, t_end, x[10:13], x[13:16], *noise)
        for key in ("dt", "dq", "dp", "dv", "cov", "dq_dbg", "dp_dbg", "dp_dba", "dv_dbg", "dv_dba"):
            assert np.array_equal(d[key], ref[key]), (k, key)
        # t_end is frame k + 1's time, where factor k + 1's samples start: it takes t_end, except after the newest
        fr, st, _ = to.trajectory([t_end], frames, factors, noise)
        if k + 1 < len(factors):
            assert fr[0] == k + 1 and np.array_equal(st[0], frames[k + 1])
        else:
            assert fr[0] == k and np.array_equal(st[0], sco.predict(x, ref))


def test_a_prefix_is_the_integration_of_the_samples_before_it():
    frames, factors, noise, _ = _window()
    s, t_end = factors[2]
    x = frames[2]
    for j in (0, 1, 7, len(s) - 1):
        for t in (s[j, 0], s[j, 0] + 0.3 * ((s[j + 1, 0] if j + 1 < len(s) else t_end) - s[j, 0])):
            d = to.delta(s, t, x[10:13], x[13:16], noise)
            if t == s[0, 0]:
                assert d["dt"] == 0.0
                continue
            assert abs(d["dt"] - (t - s[0, 0])) < 1e-12
            if j >= 7:                                 # (shorter prefixes have no sqrt_inv_cov for integrate to form)
                ref = imu_oracle.integrate(s[:j + 1], t, x[10:13], x[13:16], *noise)
                assert np.array_equal(d["dp"], ref["dp"]) and np.array_equal(d["cov"], ref["cov"])


def test_factor_selection_at_gaps_boundaries_and_factors_without_samples():
    frames, factors, noise, _ = _window(N=7)
    # factor 1 starts 5e-6 s after frame 1 (the prepend rule's gap), factor 3 holds no samples
    s1, t1 = factors[1]
    s1 = s1.copy()
    s1[0, 0] += 5e-6
    factors[1] = (s1, t1)
    factors[3] = (None, factors[3][1])
    t_end = [f[1] for f in factors]
    start = [None if f[0] is None else f[0][0, 0] for f in factors]
    cases = [
        (start[0] - 1e-3, -1),                       # before the first sample
        (start[0], 0),
        (0.5 * (start[0] + t_end[0]), 0),
        (t_end[0], 0),                               # t_end of factor 0 = frame 1's time, before factor 1's s_0
        (t_end[0] + 2e-6, 0),                        # the gap: factor 1 holds samples, so factor 0 runs on
        (start[1], 1),
        (t_end[1] - 1e-6, 1),
        (t_end[1], 2),                               # frame 2's time: factor 2 starts there
        (t_end[2], 2),                               # factor 3 holds none: factor 2 stops at its t_end
        (t_end[2] + 1e-6, -1),
        (0.5 * (t_end[2] + t_end[3]), -1),           # over the factor without samples
        (start[4], 4),
        (t_end[5], 5),                               # the newest frame's time
        (t_end[5] + 1e-6, -1),                       # after the newest frame
    ]
    for t, k in cases:
        assert to.factor_of(t, factors) == k, (t, k)
    fr, st, cov = to.trajectory([t for t, _ in cases], frames, factors, noise, np.zeros((7, 15, 15)))
    assert list(fr) == [k for _, k in cases]
    out = fr < 0
    assert np.all(st[out] == 0.0) and np.isnan(cov[out]).all() and np.isfinite(cov[~out]).all()
    # in the gap the last increment runs past t_end
    x = frames[0]
    ref = imu_oracle.integrate(factors[0][0], t_end[0] + 2e-6, x[10:13], x[13:16], *noise)
    assert np.array_equal(st[4], sco.predict(x, ref))
