"""pvio_b200_batch_window_trajectory: the state of solved inertial slots with kept IMU samples and a prior at any time
inside the window, against oracle/trajectory_oracle.py with each frame's marginal covariance from cov_oracle; the
frame-time and t_end properties, the uncovered times, the numeric status, batching, no side effects, rejections and the
launch count.

The device integrates with fused multiply-adds, as pvio_b200_preintegrate and the re-integration before a solve do, so
states are held to the oracle at 1e-12 (the bar test_gpu_batch_window_imu.py holds the records to), and bit for bit
to the device's own quantities: the frame states at each factor's first sample."""
import ctypes as C

import numpy as np
import pytest

from oracle import cov_oracle
from oracle import imu_stream_cov_oracle as sco
from oracle import trajectory_oracle as to
from pvio_b200 import _lib, imu
from pvio_b200.batch_window import BatchWindows, Imu
from pvio_b200.bundle_adjustor import BundleAdjustor, PvioB200Error
from synthetic import synth
from test_gpu_batch_window_covariance import BAR_FP64, _err, _feed, _repack, _tracks

pytestmark = pytest.mark.gpu
EINVAL = f"error {_lib.EINVAL}"
# (N, seed, factors without samples, factors whose first sample lies 5e-6 s after their frame)
SLOTS = [(5, 960, (), ()), (7, 961, (3,), (1,)), (9, 962, (), (2, 5))]


def _seat(bw, slot, N, seed, skip, shift, one=()):
    w, st, truth = synth.make_cfg3(N=N, M=120, seed=seed)
    model = _feed(bw, slot, w, st, _tracks(w, planes=False))
    factors, recs = [], []
    for k in range(N - 1):
        s, t = truth.imu_factors[k][0].copy(), truth.imu_factors[k][1]
        if k in shift:
            s[0, 0] += 5e-6
        if k in one:
            s = s[:1]
        factors.append((None, t) if k in skip else (s, t))
        if k not in skip:
            recs.append(Imu(slot, k + 1, s, t, truth.imu_noise))
    bw.set_imu(recs)
    return dict(w=w, model=model, factors=factors, noise=truth.imu_noise)


def _times(factors):
    ts = []
    for s, t_end in factors:
        if s is None:
            continue
        ts += list(s[:, 0]) + list(0.5 * (s[1:, 0] + s[:-1, 0])[::7]) + [t_end, t_end + 2e-6]
    first = min(s[0, 0] for s, _ in factors if s is not None)
    ts += [first - 1e-3, factors[-1][1] + 1e-3, 0.5 * (factors[-1][1] + factors[-2][1])]
    return np.sort(np.array(ts))


@pytest.fixture(scope="module")
def seq():
    ba = BundleAdjustor(max_windows=136, max_frames=9, max_landmarks=130, max_obs=1500)
    bw = BatchWindows(ba)
    info = [_seat(bw, j, *c) for j, c in enumerate(SLOTS)]
    info.append(_seat(bw, 3, 6, 963, (), (), one=(2,)))           # a one-sample factor: H is not positive definite
    bw.solve([0, 1, 2, 3], max_iterations=4)
    yield ba, bw, info
    ba.close()


def _sigma(bw, slot, inf):
    """each frame's marginal covariance from cov_oracle at the slot's state"""
    d = bw.download([slot], 600)[0]
    wr, sr, _ = _repack(inf["w"], d, inf["model"], bw.imu_records([slot])[0], list(inf["w"].frame_fixed))
    N = wr.N
    joint, _, _ = cov_oracle.covariance(wr, sr, list(range(N)), [], refine=True)
    return d["frames"], np.array([joint[15 * f:15 * f + 15, 15 * f:15 * f + 15] for f in range(N)])


def test_states_and_covariances_against_the_oracle(seq):
    ba, bw, info = seq
    for j in range(3):
        inf = info[j]
        ts = _times(inf["factors"])
        out = bw.trajectory([j], [ts], covariance=True)[0]
        assert out["status"] == _lib.OK
        frames, Sig = _sigma(bw, j, inf)
        fr, st, cov = to.trajectory(ts, frames, inf["factors"], inf["noise"], Sig)
        assert np.array_equal(out["frame"], fr), j
        cov_k = out["state_cov"]
        on = fr >= 0
        assert np.all(out["states"][~on] == 0.0) and np.isnan(cov_k[~on]).all()
        e = np.abs(out["states"][on] - st[on]) / (1.0 + np.abs(st[on]))
        worst = max(_err(c, r) for c, r in zip(cov_k[on], cov[on]))
        print(f"slot {j}: {on.sum()} times, state error {e.max():.2e}, covariance error {worst:.2e}")
        assert e.max() < 1e-12
        assert worst < BAR_FP64[0]
        assert np.array_equal(cov_k, np.transpose(cov_k, (0, 2, 1)), equal_nan=True)
        # at each factor's first sample: the frame's state and the frame's block of batch_window_covariance, bit for bit
        for k, (s, t_end) in enumerate(inf["factors"]):
            if s is None:
                continue
            r = bw.trajectory([j], [[s[0, 0]]], covariance=True)[0]
            assert r["frame"][0] == k and np.array_equal(r["states"][0], frames[k]), (j, k)
            blk = bw.covariance([j], [[k]], [[]])[0]["cov"]
            assert np.array_equal(r["state_cov"][0], blk), (j, k)


def test_t_end_is_the_full_factor_and_uncovered_times(seq):
    ba, bw, info = seq
    for j in range(3):
        inf = info[j]
        frames = bw.download([j], 600)[0]["frames"]
        F = inf["factors"]
        for k, (s, t_end) in enumerate(F):
            if s is None:
                continue
            if not (k + 1 == len(F) or F[k + 1][0] is None or F[k + 1][0][0, 0] > t_end):
                continue                                       # frame k + 1's factor takes t_end
            x = frames[k]
            rec = imu.preintegrate(ba, [(s, t_end, x[10:13], x[13:16])], inf["noise"])[0]
            d = dict(dt=rec[0], dq=rec[1:5], dp=rec[5:8], dv=rec[8:11])
            got = bw.trajectory([j], [[t_end]])[0]
            assert got["frame"][0] == k
            ref = sco.predict(x, d)
            assert np.max(np.abs(got["states"][0] - ref) / (1.0 + np.abs(ref))) < 1e-12, (j, k)
        first = min(s[0, 0] for s, _ in F if s is not None)
        probe = [first - 1e-6, F[-1][1] + 1e-6]
        for k, (s, t_end) in enumerate(F):
            if s is None:
                probe.append(0.5 * (F[k - 1][1] + t_end))     # over a factor without samples
        got = bw.trajectory([j], [sorted(probe)], covariance=True)[0]
        assert np.all(got["frame"] == -1) and np.all(got["states"] == 0.0) and np.isnan(got["state_cov"]).all()


def test_numeric_status(seq):
    ba, bw, info = seq
    inf = info[3]
    assert bw.covariance([3], [[0]], [[]])[0]["status"] == _lib.ENUMERIC
    ts = _times(inf["factors"])
    r = bw.trajectory([3, 0], [ts, [info[0]["factors"][1][0][3, 0]]], covariance=True)
    assert r[0]["status"] == _lib.ENUMERIC and np.isnan(r[0]["state_cov"]).all()
    assert np.all(np.isfinite(r[0]["states"][r[0]["frame"] >= 0]))
    assert r[1]["status"] == _lib.OK and np.isfinite(r[1]["state_cov"]).all()


def test_batches_give_the_bits_of_single_records_and_change_nothing(seq):
    ba, bw, info = seq
    blobs = bw.save([0, 1, 2])
    W = 132
    slots = list(range(4, 4 + W))
    bw.restore(slots, [blobs[i % 3] for i in range(W)])
    ts = [_times(info[i % 3]["factors"])[::(1 + i % 5)] for i in range(W)]
    before = bw.save(slots[:8] + [0, 1, 2, 3])
    for n in (1, 8, W):
        for cov in (False, True):
            L = ba.kernel_launches
            many = bw.trajectory(slots[:n], ts[:n], covariance=cov)
            assert ba.kernel_launches - L == (4 if cov else 1), (n, cov)
            for i in range(n):
                one = bw.trajectory([slots[i]], [ts[i]], covariance=cov)[0]
                for key in one:
                    assert np.array_equal(np.asarray(one[key]), np.asarray(many[i][key]), equal_nan=True), (n, i, key)
    assert bw.save(slots[:8] + [0, 1, 2, 3]) == before


def test_rejections_leave_every_output(seq):
    ba, bw, info = seq
    assert C.sizeof(_lib.CWindowTrajectory) == 48
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
        rc = handle.lib.pvio_b200_batch_window_trajectory(handle.h, 2 if n is None else n, recs)
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
    assert vis.lib.pvio_b200_batch_window_trajectory(vis.h, 1, recs) == _lib.EINVAL     # a visual-only slot
    assert bw.save([0, 1, 2, 3]) == before
    with pytest.raises(PvioB200Error, match=EINVAL):
        bw.trajectory([0], [ts[::-1]])
    vis.close()
