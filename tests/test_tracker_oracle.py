"""The CPU oracles of pvio_b200_batch_window_track_frame: tracker_oracle.keyframe_check (sliding_window_tracker.cpp:
255-296) on hand-built parallax lists, and tracker_oracle.predict (preintegrator.cpp:102-109) against its closed
form."""
import numpy as np
import pytest

from oracle import imu_oracle, lie, tracker_oracle

ID = np.array([0.0, 0.0, 0.0, 1.0])
FX, FY, CX, CY = 100.0, 100.0, 320.0, 240.0


def _check(pars, skipped=0, dq=ID):
    """keyframe_check with identity extrinsics and rotation: each pair's parallax is the plain pixel distance given"""
    pars = np.asarray(pars, dtype=np.float64)
    z_i = np.zeros((len(pars), 2))
    z_j = np.stack([pars / FX, np.zeros(len(pars))], axis=1)
    return tracker_oracle.keyframe_check(z_i, z_j, dq, ID, ID, FX, FY, CX, CY, skipped)


def test_fewer_than_50_pairs_is_a_keyframe():
    kf, par, m, sk = _check(np.full(49, 1.0), skipped=3)
    assert kf and np.isnan(par) and m == 49 and sk == 0
    kf, par, m, sk = _check(np.full(50, 1.0), skipped=3)
    assert not kf and par == pytest.approx(1.0) and m == 50 and sk == 4


@pytest.mark.parametrize("m", [50, 51, 99])
def test_the_percentile_index_is_m_times_4_div_5(m):
    vals = np.arange(m) + 0.25
    rng = np.random.default_rng(m)
    _, par, got_m, _ = _check(rng.permutation(vals))
    assert got_m == m
    assert par == pytest.approx(vals[m * 4 // 5], abs=1e-9)
    assert m * 4 // 5 == {50: 40, 51: 40, 99: 79}[m]


def test_the_threshold_is_strictly_above_50_px():
    pars = np.concatenate([np.full(40, 1.0), np.full(10, 50.0)])          # element 40 of 50 is exactly 50 px
    kf, par, _, sk = _check(pars)
    assert par == 50.0 and not kf and sk == 1
    pars[40:] = 50.0 + 1e-9
    kf, par, _, sk = _check(pars)
    assert par > 50.0 and kf and sk == 0


def test_the_skipped_counter_forces_a_keyframe_after_10():
    low = np.full(60, 5.0)
    assert _check(low, skipped=9)[3] == 10 and not _check(low, skipped=9)[0]
    kf, _, _, sk = _check(low, skipped=10)                                 # 11 > 10: forced, then reset
    assert kf and sk == 0
    kf, _, _, sk = _check(low, skipped=11)
    assert kf and sk == 0


def test_q7_frame_i_before_the_newest_frame_uses_the_new_frames_rotation():
    """quirk Q7: with frame_i = N - 2, qij still comes from the new frame's own delta q (rotating from the newest
    frame), so a rotation between frame_i and the newest frame shows up as parallax"""
    rng = np.random.default_rng(7)
    x = rng.normal(size=(60, 3)) + np.array([0.0, 0.0, 6.0])                # points in the camera of frame_i
    q_in = lie.expmap(np.array([0.0, 0.08, 0.0]))                           # frame_i -> newest (not in the record)
    dq = lie.expmap(np.array([0.02, 0.0, 0.0]))                             # newest -> new frame: the record's
    q_ij = lie.qmul(q_in, dq)
    y = np.array([lie.qrot(lie.qconj(q_ij), p) for p in x])                 # the same points seen from the new frame
    z_i, z_j = x[:, :2] / x[:, 2:], y[:, :2] / y[:, 2:]
    kf, par, m, _ = tracker_oracle.keyframe_check(z_i, z_j, dq, ID, ID, FX, FY, CX, CY, 0)
    _, par_true, _, _ = tracker_oracle.keyframe_check(z_i, z_j, q_ij, ID, ID, FX, FY, CX, CY, 0)
    assert m == 60 and par_true < 1e-9                                      # the full rotation explains every pair
    assert par > 5.0                                                        # the reference's qij leaves 0.08 rad of it


def test_predict_matches_the_closed_form_for_constant_acceleration():
    a, T, n = np.array([0.3, -0.2, 9.9]), 0.1, 20
    t = np.arange(n) * (T / n)
    smp = np.concatenate([t[:, None], np.zeros((n, 3)), np.tile(a, (n, 1))], axis=1)
    cov = np.eye(3) * 1e-4
    rec = imu_oracle.record(imu_oracle.integrate(smp, T, np.zeros(3), np.zeros(3), cov, cov, cov, cov),
                            np.zeros(3), np.zeros(3))
    x = np.concatenate([ID, [1.0, 2.0, 3.0], [0.5, -0.1, 0.2], np.full(3, 1e-3), np.full(3, -2e-3)])
    y = tracker_oracle.predict(x, rec)
    g = np.array([0.0, 0.0, -9.80665])
    assert np.allclose(y[0:4], ID, atol=0, rtol=0)
    assert np.abs(y[7:10] - (x[7:10] + (g + a) * T)).max() <= 1e-12
    assert np.abs(y[4:7] - (x[4:7] + x[7:10] * T + 0.5 * (g + a) * T * T)).max() <= 1e-12
    assert np.array_equal(y[10:16], x[10:16])
