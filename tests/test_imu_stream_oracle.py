"""oracle/imu_stream_oracle.py against hand-built streams: the synchronisation of gyroscope and accelerometer readings
(core.cpp:59-107), the sorting of samples into camera frames (:129-141), the prepend rule (feature_tracker.cpp:78-84),
the lockstep rule, and the IMU-rate pose (:143-164) against closed-form motion and the output extrinsic."""
import math

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from oracle import imu_stream_oracle as so
from oracle.imu_stream_oracle import ACCELEROMETER as A, CAMERA as C, GYROSCOPE as G


def _run(events, stream=None):
    """feeds every event (re-pushing after each release); returns the stream, all poses and all released frames"""
    s = stream or so.Stream()
    poses, frames, ev = [], [], list(events)
    while ev:
        p, n, rel = s.push(ev)
        poses += p
        frames += rel
        ev = ev[n:]
    return s, poses, frames


def _w(t):
    return (0.1 + t, -0.2 * t, 0.3 - t * t)


def _a(t):
    return (0.5 * t, 9.8 + t, -0.1)


def test_equal_stamps_in_either_arrival_order_give_the_same_samples():
    ts = [0.005 * k for k in range(12)]
    gyro_first, acc_first = [], []
    for t in ts:
        gyro_first += [(G, t, *_w(t)), (A, t, *_a(t))]
        acc_first += [(A, t, *_a(t)), (G, t, *_w(t))]
    for evs in (gyro_first, acc_first):
        s, _, _ = _run([(C, 0.03, 0, 0, 0)] + evs)
        got = [(x[0], *x[1], *x[2]) for x in s.frontal_imus]
        # gyroscope first: the sample at a reading's own stamp; accelerometer first: from the second stamp on
        # (the first accelerometer reading finds no gyroscope reading and is ignored)
        want = [(t, *_w(t), *_a(t)) for t in (ts if evs is gyro_first else ts[1:])]
        np.testing.assert_allclose(np.array(got), np.array(want), rtol=0, atol=1e-15)


def test_separate_rates_interpolate_the_gyroscope_at_accelerometer_times():
    evs = []
    for k in range(20):
        evs.append((G, 0.01 * k, *_w(0.01 * k)))
        evs.append((A, 0.01 * k + 0.004, *_a(0.01 * k + 0.004)))
    s, _, _ = _run(evs)
    rows = np.array([(x[0], *x[1], *x[2]) for x in s.frontal_imus])
    assert len(rows) == 19                              # the last accelerometer reading waits for a later gyroscope one
    tg = 0.01 * np.arange(20)
    for j in range(3):
        np.testing.assert_allclose(rows[:, 1 + j], np.interp(rows[:, 0], tg, [_w(t)[j] for t in tg]), atol=1e-15)
    np.testing.assert_array_equal(rows[:, 4:7], np.array([_a(t) for t in rows[:, 0]]))


def test_accelerometer_readings_before_any_gyroscope_are_ignored():
    s, _, _ = _run([(A, 0.0, *_a(0)), (A, 0.01, *_a(0.01)), (G, 0.02, *_w(0.02)), (A, 0.015, *_a(0.015))])
    assert not s.frontal_imus and not s.accelerometers   # 0.015 is before the only gyroscope reading too


def test_a_gyroscope_reading_older_than_the_accelerometer_queue_clears_the_gyroscopes():
    s, _, _ = _run([(G, 0.0, 1, 1, 1), (A, 0.5, *_a(0.5)), (G, 0.3, 2, 2, 2), (G, 0.6, 5, 5, 5)])
    (t, w, _), = s.frontal_imus
    lam = (0.5 - 0.3) / (0.6 - 0.3)                      # from 0.3, not 0.0
    assert t == 0.5 and w == tuple(2 + lam * (5 - 2) for _ in range(3))


def test_one_sample_releases_two_frames_and_the_empty_one_takes_the_previous_last_sample():
    evs = [(G, 0.0, *_w(0)), (C, 0.1, 0, 0, 0), (C, 0.2, 0, 0, 0), (A, 0.05, *_a(0.05)), (A, 0.25, *_a(0.25)),
           (G, 0.3, *_w(0.3)), (A, 0.28, *_a(0.28))]
    s = so.Stream()
    _, n, rel = s.push(evs)
    assert n == 6                                        # the gyroscope reading that released both frames
    (t1, r1), (t2, r2) = rel
    assert (t1, t2) == (0.1, 0.2) and len(r1) == 1 and r1[0][0] == 0.05
    assert len(r2) == 1 and r2[0][0] == 0.1 and r2[0][1:] == r1[0][1:]     # prepended at the previous frame's time


@pytest.mark.parametrize("gap, prepended", [(2e-5, True), (0.5e-5, False)])
def test_prepend_rule_threshold(gap, prepended):
    t0 = 1.0
    evs = [(G, 0.99, *_w(0.99)), (A, 0.99, *_a(0.99)), (C, t0, 0, 0, 0), (C, t0 + 0.05, 0, 0, 0),
           (G, t0 + gap, *_w(t0 + gap)), (A, t0 + gap, *_a(t0 + gap)),
           (G, t0 + 0.06, *_w(t0 + 0.06)), (A, t0 + 0.06, *_a(t0 + 0.06))]
    _, _, frames = _run(evs)
    (_, r1), (_, r2) = frames
    assert r1[-1][0] == 0.99
    assert len(r2) == (2 if prepended else 1)
    if prepended:
        assert r2[0] == [t0] + r1[-1][1:]


def test_no_state_gives_the_invalid_pose_and_a_cleared_state_again():
    evs = [(G, 0.01 * k, *_w(0.01 * k)) for k in range(3)]
    s, poses, _ = _run(evs)
    assert all(p == (0.0,) * 7 for p in poses)
    st = (0, 0, 0, 1, 1, 2, 3, 0, 0, 0, 0, 0, 0, 0, 0, 0)
    p, _, _ = s.push([(G, 0.03, 0, 0, 0)], state=(0.0, st))
    assert p[0][3] == 1.0 and p[0][4:] == (1.0, 2.0, 3.0)
    p, _, _ = s.push([(G, 0.04, 0, 0, 0)], clear=True)
    assert p[0] == (0.0,) * 7


def test_state_drops_older_samples_and_an_early_event_propagates_less():
    evs = []
    for k in range(10):
        evs += [(G, 0.01 * k, *_w(0.01 * k)), (A, 0.01 * k, *_a(0.01 * k))]
    s, _, _ = _run(evs)
    st = (0, 0, 0, 1) + (0.0,) * 12
    p_late, _, _ = s.push([(G, 0.1, *_w(0.1))], state=(0.045, st))
    assert all(x[0] > 0.045 for x in s.frontal_imus)
    p_early, _, _ = s.push([(C, 0.05, 0, 0, 0)])           # a camera stamp behind the IMU: samples 0.05 .. only
    ref = [0.045, st[0:4], st[4:7], st[7:10], st[10:13], st[13:16]]
    ref = so.propagate(ref, 0.05, _w(0.05), _a(0.05))
    assert p_early[0][:4] == ref[1] and p_early[0][4:] == ref[2]
    assert p_late[0] != p_early[0]


def test_constant_rate_rotation_and_free_motion_follow_the_closed_form():
    """world acceleration zero: each accelerometer reading is gravity's reaction in the body at the start of its
    interval, the rate constant about a fixed axis: q(t) = exp(w t), p(t) = p0 + v0 t"""
    w = np.array([0.3, -0.2, 0.5])
    v0, p0 = np.array([1.0, -0.5, 0.25]), np.array([2.0, 0.0, -1.0])
    s = so.Stream()
    dt, n = 0.005, 200
    s.set_state(0.0, (0, 0, 0, 1, *p0, *v0, 0, 0, 0, 0, 0, 0))
    pose = None
    for k in range(1, n + 1):
        t = k * dt
        R_prev = Rotation.from_rotvec(w * (t - dt))
        a = R_prev.inv().apply([0.0, 0.0, so.GRAVITY])
        s.gyroscope(t, *w)
        pose = s.accelerometer(t, *a)
    T = n * dt
    q_want = Rotation.from_rotvec(w * T).as_quat()
    assert min(np.abs(np.array(pose[:4]) - q_want).max(), np.abs(np.array(pose[:4]) + q_want).max()) < 1e-12
    np.testing.assert_allclose(pose[4:], p0 + v0 * T, atol=1e-9)


def test_output_extrinsic():
    q_ob = Rotation.from_rotvec([0.1, 0.2, -0.3]).as_quat()
    p_ob = np.array([0.05, -0.02, 0.1])
    q_s = Rotation.from_rotvec([-0.4, 0.3, 0.2])
    p_s = np.array([1.0, 2.0, 3.0])
    s = so.Stream(q_ob, p_ob)
    s.set_state(0.0, (*q_s.as_quat(), *p_s) + (0.0,) * 9)
    pose = s.camera(0.0)                               # no samples: the state itself
    np.testing.assert_allclose((q_s * Rotation.from_quat(q_ob)).as_quat(), pose[:4], atol=1e-15)
    np.testing.assert_allclose(p_s + q_s.apply(p_ob), pose[4:], atol=1e-15)


def test_expmap_is_the_lie_oracles_to_rounding():
    from oracle import lie
    rng = np.random.default_rng(3)
    for u in rng.normal(size=(50, 3)) * 0.05:
        np.testing.assert_allclose(so.expmap(tuple(u)), lie.expmap(u), rtol=0, atol=4e-16)
    assert so.expmap((0.0, 0.0, 0.0)) == (0.0, 0.0, 0.0, 1.0) and math.isfinite(so.expmap((1e-300, 0, 0))[0])
