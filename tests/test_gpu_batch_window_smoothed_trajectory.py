"""pvio_b200_batch_window_smoothed_trajectory: the state of solved inertial slots conditioned on both frames around each
time, against trajectory_smoothing_oracle.smoothed with the window's joint frame covariance from cov_oracle; the
endpoint properties, the factor each time is taken by (the forward call's, or -2 on a one-sample factor), the gap rule,
the numeric status, batching, no side effects, rejections and the launch count.

The slots are those of test_gpu_batch_window_trajectory.py: solved cfg3 windows with kept samples and a prior, some with
factors without samples or with first samples 5e-6 s after their frame, and one with a one-sample factor."""
import ctypes as C

import numpy as np
import pytest

from oracle import cov_oracle
from pvio_b200 import _lib
from pvio_b200.batch_window import BatchWindows
from pvio_b200.bundle_adjustor import BundleAdjustor, PvioB200Error
from synthetic import synth
from test_gpu_batch_window_covariance import BAR_FP64, _err, _repack
from test_gpu_batch_window_trajectory import SLOTS, _seat, _times
import trajectory_smoothing_oracle as tso

pytestmark = pytest.mark.gpu
EINVAL = f"error {_lib.EINVAL}"


@pytest.fixture(scope="module")
def seq():
    ba = BundleAdjustor(max_windows=136, max_frames=9, max_landmarks=130, max_obs=1500)
    bw = BatchWindows(ba)
    info = [_seat(bw, j, *c) for j, c in enumerate(SLOTS)]
    info.append(_seat(bw, 3, 6, 963, (), (), one=(2,)))           # a one-sample factor: H is not positive definite
    bw.solve([0, 1, 2, 3], max_iterations=4)
    yield ba, bw, info
    ba.close()


def _joint(bw, slot, inf):
    """the slot's frames and the joint covariance of all of them from cov_oracle at the slot's state"""
    d = bw.download([slot], 600)[0]
    wr, sr, _ = _repack(inf["w"], d, inf["model"], bw.imu_records([slot])[0], list(inf["w"].frame_fixed))
    joint, _, _ = cov_oracle.covariance(wr, sr, list(range(wr.N)), [], refine=True)
    return d["frames"], joint


def _rel(a, b):
    return np.abs(a - b) / (1.0 + np.abs(b))


def test_states_and_covariances_against_the_oracle(seq):
    ba, bw, info = seq
    for j in range(3):
        inf = info[j]
        ts = _times(inf["factors"])
        out = bw.trajectory([j], [ts], covariance=True, smoothed=True)[0]
        fwd = bw.trajectory([j], [ts])[0]
        assert out["status"] == _lib.OK
        assert np.array_equal(out["frame"], fwd["frame"]), j
        frames, joint = _joint(bw, j, inf)
        fr, st, cov = tso.smoothed(ts, frames, inf["factors"], inf["noise"], joint)
        assert np.array_equal(out["frame"], fr), j
        on = fr >= 0
        assert np.all(out["states"][~on] == 0.0) and np.isnan(out["state_cov"][~on]).all()
        e = _rel(out["states"][on], st[on])
        worst = max(_err(c, r) for c, r in zip(out["state_cov"][on], cov[on]))
        print(f"slot {j}: {on.sum()} times, state error {e.max():.2e}, covariance error {worst:.2e}")
        assert e.max() < 1e-11
        assert worst < BAR_FP64[0]
        sc = out["state_cov"]
        assert np.array_equal(sc, np.transpose(sc, (0, 2, 1)), equal_nan=True)
        # the states without covariances are the same bits
        assert np.array_equal(bw.trajectory([j], [ts], smoothed=True)[0]["states"], out["states"])


def test_endpoints_are_the_frames(seq):
    ba, bw, info = seq
    for j in range(3):
        F = info[j]["factors"]
        frames = bw.download([j], 600)[0]["frames"]
        for k, (s, t_end) in enumerate(F):
            if s is None:
                continue
            r = bw.trajectory([j], [[s[0, 0]]], smoothed=True)[0]
            assert r["frame"][0] == k and np.array_equal(r["states"][0], frames[k]), (j, k)
            if not (k + 1 == len(F) or F[k + 1][0] is None or F[k + 1][0][0, 0] > t_end):
                continue                                       # frame k + 1's factor takes t_end
            r = bw.trajectory([j], [[t_end]], smoothed=True)[0]
            assert r["frame"][0] == k
            y = r["states"][0].copy()
            y[0:4] *= np.sign(y[3] * frames[k + 1][3])
            assert _rel(y, frames[k + 1]).max() < 1e-12, (j, k)


def test_one_sample_factor_and_numeric_status(seq):
    ba, bw, info = seq
    inf = info[3]
    assert bw.covariance([3], [[0]], [[]])[0]["status"] == _lib.ENUMERIC
    ts = _times(inf["factors"])
    fwd = bw.trajectory([3], [ts])[0]
    r = bw.trajectory([3, 0], [ts, [info[0]["factors"][1][0][3, 0]]], covariance=True, smoothed=True)
    assert r[0]["status"] == _lib.ENUMERIC and np.isnan(r[0]["state_cov"]).all()
    two = fwd["frame"] == 2
    assert two.any()
    assert np.all(r[0]["frame"][two] == -2) and np.all(r[0]["states"][two] == 0.0)
    assert np.array_equal(r[0]["frame"][~two], fwd["frame"][~two])
    assert np.all(np.isfinite(r[0]["states"][r[0]["frame"] >= 0]))
    assert r[1]["status"] == _lib.OK and np.isfinite(r[1]["state_cov"]).all()
    frames = bw.download([3], 600)[0]["frames"]
    fr, st, _ = tso.smoothed(ts, frames, inf["factors"], inf["noise"])
    assert np.array_equal(r[0]["frame"], fr)
    on = fr >= 0
    assert _rel(r[0]["states"][on], st[on]).max() < 1e-11


def test_batches_give_the_bits_of_single_records_and_change_nothing(seq):
    ba, bw, info = seq
    blobs = bw.save([0, 1, 2])
    W = 132
    slots = list(range(4, 4 + W))
    bw.restore(slots, [blobs[i % 3] for i in range(W)])
    ts = [_times(info[i % 3]["factors"])[::(1 + i % 5)] for i in range(W)]
    probe = slots[:8] + [0, 1, 2, 3]
    before = bw.save(probe)
    d0 = bw.download(probe, 600)
    f0 = bw.trajectory(probe, [ts[0]] * len(probe), covariance=True)
    for n in (1, 8, W):
        for cov in (False, True):
            L = ba.kernel_launches
            many = bw.trajectory(slots[:n], ts[:n], covariance=cov, smoothed=True)
            assert ba.kernel_launches - L == (4 if cov else 1), (n, cov)
            for i in range(n):
                one = bw.trajectory([slots[i]], [ts[i]], covariance=cov, smoothed=True)[0]
                for key in one:
                    assert np.array_equal(np.asarray(one[key]), np.asarray(many[i][key]), equal_nan=True), (n, i, key)
    assert bw.save(probe) == before
    d1 = bw.download(probe, 600)
    for a, b in zip(d0, d1):
        for key in a:
            assert np.array_equal(np.asarray(a[key]), np.asarray(b[key]), equal_nan=True), key
    f1 = bw.trajectory(probe, [ts[0]] * len(probe), covariance=True)
    for a, b in zip(f0, f1):
        for key in a:
            assert np.array_equal(np.asarray(a[key]), np.asarray(b[key]), equal_nan=True), key


def test_rejections_leave_every_output(seq):
    ba, bw, info = seq
    ts = _times(info[0]["factors"])
    vis = BundleAdjustor(max_windows=1, max_frames=6, max_landmarks=100, max_obs=600)
    w, st, _ = synth.make_cfg2(N=5, M=40)
    vb = BatchWindows(vis)
    vb.reset(0, w)

    def run(spoil, handle=ba, n=None):
        k = len(ts)
        t = ts.copy()
        outs = [np.full((k, 16), 7.0), np.full((k, 225), 7.0), np.full(k, 7, dtype=np.int32)]
        recs = (_lib.CWindowTrajectory * 2)()
        for r, s in zip(recs, (0, 1)):
            r.slot, r.n_times, r.status = s, k, 99
            _lib.set_ptrs(r, times=t, states=outs[0], state_cov=outs[1], frame=outs[2])
        spoil(recs, t)
        rc = handle.lib.pvio_b200_batch_window_smoothed_trajectory(handle.h, 2 if n is None else n, recs)
        assert rc == _lib.EINVAL
        assert np.all(outs[0] == 7.0) and np.all(outs[1] == 7.0) and np.all(outs[2] == 7)
        assert recs[0].status == 99 and recs[1].status == 99

    def setf(**kw):
        def f(recs, t):
            for k, v in kw.items():
                setattr(recs[1], k, v)
        return f

    def nan_time(recs, t):
        t[5] = np.nan

    def decreasing(recs, t):
        t[5], t[6] = t[6], t[5]

    before = bw.save([0, 1, 2, 3])
    run(lambda r, t: None, n=-1)
    run(setf(slot=136))
    run(setf(slot=-1))
    run(setf(slot=0))                                      # named twice
    run(setf(n_times=-1))
    run(setf(times=None))
    run(setf(states=None))
    run(setf(frame=None))
    run(nan_time)
    run(decreasing)
    recs = (_lib.CWindowTrajectory * 1)()
    recs[0].slot, recs[0].n_times = 0, 0
    assert vis.lib.pvio_b200_batch_window_smoothed_trajectory(vis.h, 1, recs) == _lib.EINVAL     # a visual-only slot
    assert bw.save([0, 1, 2, 3]) == before
    with pytest.raises(PvioB200Error, match=EINVAL):
        bw.trajectory([0], [ts[::-1]], smoothed=True)
    assert ba.lib.pvio_b200_batch_window_smoothed_trajectory(ba.h, 0, None) == 0
    vis.close()
