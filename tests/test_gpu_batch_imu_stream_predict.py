"""pvio_b200_batch_imu_stream_set_covariance / pvio_b200_batch_imu_stream_predict: predicted poses against
oracle/imu_stream_oracle.py bit for bit (264 sequences of mixed stream shapes, queried before the state, on and between
sample stamps, beyond the last sample, with the state's drop pending and done), covariances against
oracle/imu_stream_cov_oracle.py (DIRECT and FACTOR seeds, and end to end from a resident inertial slot's window
covariance through track_frame), the call's read-only-ness, the seed's validity, rejections and launch counts.  The
oracle is given the device's sin / cos of the same arguments (torch on the same GPU), as in test_gpu_batch_imu_stream."""
import collections
import math

import numpy as np
import pytest

from oracle import imu_oracle, lie
from oracle import imu_stream_cov_oracle as co
from oracle import imu_stream_oracle as so
from pvio_b200 import _lib
from pvio_b200.bundle_adjustor import BundleAdjustor, PvioB200Error
from pvio_b200.imu_stream import NO_COVARIANCE, NO_STATE, ImuStream, StreamRecord

pytestmark = pytest.mark.gpu
G, A, C = so.GYROSCOPE, so.ACCELEROMETER, so.CAMERA
NOISE = np.stack([np.diag([1e-4, 2e-4, 1.5e-4]), np.diag([3e-3, 2e-3, 4e-3]), np.diag([1e-7, 2e-7, 1e-7]),
                  np.diag([2e-5, 1e-5, 3e-5])]).reshape(4, 9)
COV_TOL = 1e-10


def _events(seed):
    """one sequence's arrival-ordered events over about 0.6 s: gyroscope and accelerometer at equal or different rates,
    jitter, camera stamps behind the IMU"""
    rng = np.random.default_rng(seed)
    shape = seed % 4
    g_dt = [0.005, 0.005, 0.0025, 0.004][shape]
    a_dt = g_dt if shape < 2 else [0.004, 0.005][shape - 2]
    jit = 0.0 if shape < 2 else 2e-4
    T = 0.6
    gt = np.cumsum(np.full(int(T / g_dt), g_dt) + rng.uniform(0, jit, int(T / g_dt)))
    at = gt.copy() if shape < 2 else np.cumsum(np.full(int(T / a_dt), a_dt) + rng.uniform(0, jit, int(T / a_dt)))
    cam = np.arange(0.02 + rng.uniform(0, 0.02), T, 0.05)
    lat = rng.uniform(0, 0.012) if shape == 2 else 0.0
    ev = [(t, 0 if shape != 1 else 1, (G, t, *(rng.normal(size=3) * 0.5))) for t in gt]
    ev += [(t, 1 if shape != 1 else 0, (A, t, *(np.array([0, 0, 9.8]) + rng.normal(size=3) * 0.3))) for t in at]
    ev += [(t + lat, 2, (C, t, 0.0, 0.0, 0.0)) for t in cam]
    ev.sort(key=lambda e: (e[0], e[1]))
    return np.array([e[2] for e in ev], dtype=np.float64)


def _state(rng):
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    return np.concatenate([q, rng.normal(size=3), rng.normal(size=3) * 0.5, rng.normal(size=3) * 0.01,
                           rng.normal(size=3) * 0.05])


def _spd(rng, scale=1e-3):
    a = rng.normal(size=(15, 15)) * scale
    return a @ a.T + np.eye(15) * scale * scale


class _DeviceSincos:
    """sin / cos as the device computes them: arguments not yet in the table are recorded (answered by the math
    library) and fill() computes them with torch on the GPU; a comparison runs the oracle once to record, then again"""

    def __init__(self):
        self.table, self.miss = {}, set()

    def __call__(self, x):
        if x in self.table:
            return self.table[x]
        self.miss.add(x)
        return math.sin(x), math.cos(x)

    def fill(self):
        import torch
        xs = sorted(self.miss)
        if xs:
            x = torch.tensor(xs, dtype=torch.float64, device="cuda")
            self.table.update(zip(xs, zip(torch.sin(x).cpu().tolist(), torch.cos(x).cpu().tolist())))
        self.miss.clear()


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _oracle_pose(orc, t):
    """predict_pose(t) of the oracle stream without changing it (predict_pose pops the samples up to the state)"""
    keep = collections.deque(orc.frontal_imus)
    p = orc.predict_pose(t)
    orc.frontal_imus = keep
    return np.array(p)


def _oracle_poses(orc, times, sincos):
    for _ in range(2):                                   # record the arguments, then with the device's sin / cos
        out = np.array([_oracle_pose(orc, t) for t in times]).reshape(-1, 7)
        sincos.fill()
    return out


def _oracle_cov(orc, P0, times, sincos):
    """(state_cov [k, 15, 15], pose_cov [k, 6, 6]) of the oracle stream with its state seeded with P0"""
    ts, x = orc.latest_state
    smp = list(orc.frontal_imus)
    sc, pc = [], []
    for t in times:
        st, P, _ = co.chain(ts, x, P0, smp, t, NOISE, sincos)
        sc.append(P)
        pc.append(co.pose_cov(st[1], P, orc.q_ob, orc.p_ob))
    return np.array(sc), np.array(pc)


def _close(dev, ref):
    assert np.max(np.abs(dev - ref)) <= COV_TOL * np.max(np.abs(ref))


def _symmetric(c):
    assert np.array_equal(_bits(c), _bits(np.swapaxes(c, -1, -2)))


@pytest.fixture(scope="module")
def ba():
    b = BundleAdjustor(max_windows=1, max_frames=8, max_landmarks=64, max_obs=256)
    yield b
    b.close()


def _query_times(orc, last_t):
    """before the state, at it, on the first kept sample and between the first two, on the last and beyond it, and the
    last consumed event's time"""
    ts = orc.latest_state[0]
    kept = [s[0] for s in orc.frontal_imus if s[0] > ts]
    t = [ts - 0.01, ts, last_t]
    if kept:
        t += [kept[0], kept[-1], kept[-1] + 0.013]
    if len(kept) > 1:
        t.append(0.5 * (kept[0] + kept[1]))
    return sorted(t)


def test_264_sequences_poses_bit_equal_and_covariances_to_the_oracle(ba):
    st = ImuStream(ba)
    n = 264
    rng = np.random.default_rng(11)
    slots = list(range(3, 3 + n))
    q_ob = np.tile([0.0, 0.0, 0.0, 1.0], (n, 1))
    p_ob = np.zeros((n, 3))
    for i in range(0, n, 2):                             # half the slots with an output extrinsic
        q_ob[i] = lie.qnormalized(rng.normal(size=4))
        p_ob[i] = rng.normal(size=3) * 0.1
    st.reset(slots, q_ob, p_ob)
    sincos = _DeviceSincos()
    orcs = [so.Stream(q_ob[i], p_ob[i], sincos=sincos) for i in range(n)]
    evs = [_events(s) for s in range(n)]
    pos, pending, seeds = [0] * n, [None] * n, [None] * n
    checked = dict(pose=0, drop=0, cov=0, last=0)
    while True:
        live = [i for i in range(n) if pos[i] < len(evs[i])]
        if not live:
            break
        recs, drop_only = [], []
        for i in live:
            if pending[i] is not None and rng.random() < 0.3:     # the state alone: its drop is pending at the query
                k = 0
                drop_only.append(i)
            else:
                k = 1 if rng.random() < 0.2 else int(rng.integers(1, 30))
            r = StreamRecord(slots[i], evs[i][pos[i]:pos[i] + k])
            if pending[i] is not None:
                r.set_state(*pending[i])
            recs.append(r)
        outs = st.push(recs)
        seed_rows = []
        for i, r, o in zip(live, recs, outs):
            if pending[i] is not None:
                orcs[i].set_state(*pending[i])
                seeds[i] = _spd(rng)
                seed_rows.append(i)
                pending[i] = None
            poses, nc, rel = orcs[i].push(r.events[:o["n_consumed"]])
            assert nc == o["n_consumed"]
            pos[i] += nc
            if o["frames"]:
                pending[i] = (o["frames"][-1][0], _state(rng))
        if seed_rows:
            st.set_covariance([slots[i] for i in seed_rows], [orcs[i].latest_state[0] for i in seed_rows],
                              [seeds[i] for i in seed_rows], NOISE)
        q = [i for i, o in zip(live, outs) if orcs[i].latest_state is not None]
        times = [_query_times(orcs[i], (r.events[o["n_consumed"] - 1, 1] if o["n_consumed"] else
                                        orcs[i].latest_state[0] + 0.001))
                 for i, r, o in zip(live, recs, outs) if i in set(q)]
        res = st.predict([slots[i] for i in q], times, states=True)
        by = {i: o for i, o in zip(live, outs)}
        for i, t, d in zip(q, times, res):
            assert d["status"] == 0
            ref = _oracle_poses(orcs[i], t, sincos)
            assert np.array_equal(_bits(d["poses"]), _bits(ref)), i
            assert np.array_equal(_bits(d["states"][:, 10:16]), _bits(np.tile(orcs[i].latest_state[1][10:16], (len(t), 1))))
            checked["pose"] += len(t)
            checked["drop"] += i in drop_only
            o = by[i]
            if o["n_consumed"]:
                k = t.index(recs[live.index(i)].events[o["n_consumed"] - 1, 1])
                assert np.array_equal(_bits(d["poses"][k]), _bits(o["poses"][-1]))
                checked["last"] += 1
            if rng.random() < 0.25:
                sc, pc = _oracle_cov(orcs[i], 0.5 * (seeds[i] + seeds[i].T), t, sincos)
                _close(d["state_cov"], sc)
                _close(d["pose_cov"], pc)
                _symmetric(d["state_cov"])
                _symmetric(d["pose_cov"])
                checked["cov"] += 1
    assert checked["pose"] > 5000 and checked["drop"] > 200 and checked["cov"] > 200 and checked["last"] > 1000, checked


def test_factor_seed_and_its_propagation(ba):
    """a state predicted through a factor (imu_oracle.integrate + predict) seeded FACTOR with its source frame's
    covariance: the seed itself (queried at the state time) and its propagation over new readings"""
    st = ImuStream(ba)
    rng = np.random.default_rng(12)
    n = 40
    slots = list(range(600, 600 + n))
    st.reset(slots)
    nz = co.noise_blocks(NOISE)
    sincos = _DeviceSincos()
    rows = []
    for i, s in enumerate(slots):
        src = _state(rng)
        smp = np.array([[0.005 * k, *(rng.normal(size=3) * 0.5), *(np.array([0, 0, 9.8]) + rng.normal(size=3))]
                        for k in range(int(rng.integers(1, 30)))])
        t_end = smp[-1, 0] + 0.003
        d = imu_oracle.integrate(smp, t_end, src[10:13], src[13:16], *nz)
        rec = imu_oracle.record(d, src[10:13], src[13:16])
        pred = co.predict(src, d)
        rows.append((src, t_end, rec, pred, _spd(rng, 1e-2 * (1 + i % 3))))
    st.push([StreamRecord(s).set_state(r[1], r[3]) for s, r in zip(slots, rows)])
    st.set_covariance(slots, [r[1] for r in rows], [r[4] for r in rows], NOISE, imu_records=[r[2] for r in rows])
    orcs = []
    for s, (src, t_end, rec, pred, P) in zip(slots, rows):
        o = so.Stream(sincos=sincos)
        o.set_state(t_end, pred)
        orcs.append(o)
    at_state = st.predict(slots, [[r[1]] for r in rows])
    for (src, t_end, rec, pred, P), d in zip(rows, at_state):
        _, _, _, seed = co.factor(pred[0:4], rec, P)
        _close(d["state_cov"][0], seed)
        _symmetric(d["state_cov"])
    recs = []
    for s, (src, t_end, rec, pred, P), o in zip(slots, rows, orcs):
        ev = []
        for k in range(1, 21):
            t = t_end + 0.005 * k
            ev += [(G, t, *(rng.normal(size=3) * 0.5)), (A, t, *(np.array([0, 0, 9.8]) + rng.normal(size=3)))]
        recs.append(StreamRecord(s, ev))
        o.push(ev)
    st.push(recs)
    times = [[r[1] - 0.1, r[1] + 0.0125, r[1] + 0.05, r[1] + 0.1, r[1] + 0.2] for r in rows]
    res = st.predict(slots, times, states=True)
    for (src, t_end, rec, pred, P), o, t, d in zip(rows, orcs, times, res):
        assert d["status"] == 0
        assert np.array_equal(_bits(d["poses"]), _bits(_oracle_poses(o, t, sincos)))
        seed = co.factor(pred[0:4], rec, P)[3]
        sc, pc = _oracle_cov(o, seed, t, sincos)
        _close(d["state_cov"], sc)
        _close(d["pose_cov"], pc)


def test_end_to_end_from_a_resident_inertial_slot():
    """solve -> batch_window_covariance of the newest frame -> track_frame -> SET predicted -> FACTOR seed -> predict,
    against imu_stream_cov_oracle chained from the window covariance the call returned"""
    from pvio_b200.batch_window import Edit
    from synthetic.sequence import BatchPlayer, Run
    from test_gpu_batch_window_track_frame import RUNS, _frame, _track
    runs = [Run(**RUNS[0])]
    b = BundleAdjustor(max_windows=2, max_frames=9, max_landmarks=400, max_obs=3000)
    try:
        p = BatchPlayer(b, runs)
        e = Edit(p.slots[0])
        e.remove = [p.ids[0].pop(l) for l in sorted(p.ids[0]) if runs[0].tracks[l][0][0] == runs[0].N - 1]
        p.bw.edit([e])
        p.model.edit([e])
        p.bw.solve([p.slots[0]], max_iterations=4)
        N = runs[0].N
        cov = p.bw.covariance([p.slots[0]], [[N - 1]], [[]])[0]
        assert cov["status"] == 0
        f, newest = _frame(p, 0)
        T = _track(p, 0, f, newest)[0]
        out = p.bw.track_frame([T])[0]
        noise = np.array([np.asarray(c, dtype=np.float64).reshape(9) for c in runs[0].truth.imu_noise])
        st = ImuStream(b)
        st.reset([7])
        st.push([StreamRecord(7).set_state(T.t_end, out["predicted"])])
        st.set_covariance([7], [T.t_end], [cov["cov"]], noise, imu_records=[out["imu_record"]])
        rng = np.random.default_rng(13)
        ev = []
        for k in range(1, 21):
            t = T.t_end + 0.005 * k
            ev += [(G, t, *(rng.normal(size=3) * 0.2)), (A, t, *(np.array([0, 0, 9.8]) + rng.normal(size=3) * 0.2))]
        st.push([StreamRecord(7, ev)])
        sincos = _DeviceSincos()
        o = so.Stream(sincos=sincos)
        o.set_state(T.t_end, out["predicted"])
        o.push(ev)
        times = [T.t_end, T.t_end + 0.02, T.t_end + 0.1]
        d = st.predict([7], [times])[0]
        seed = co.factor(out["predicted"][0:4], out["imu_record"], cov["cov"])[3]
        P = np.empty((len(times), 15, 15))
        for k, t in enumerate(times):
            P[k] = co.chain(T.t_end, out["predicted"], seed, list(o.frontal_imus), t,
                            noise.reshape(4, 9), sincos)[1]
        _close(d["state_cov"], P)
        assert np.array_equal(_bits(d["poses"]), _bits(_oracle_poses(o, times, sincos)))
    finally:
        b.close()


def _feed(st, slots, ev):
    while len(ev):
        o = st.push([StreamRecord(s, ev) for s in slots])
        ev = ev[o[0]["n_consumed"]:]


def _head(t0=0.0, k=12):
    ev = []
    for j in range(k):
        t = t0 + 0.005 * j
        ev += [(G, t, 0.1 + 0.01 * j, -0.2, 0.3), (A, t, 0.1, 0.05 * j, 9.8)]
    return np.array(ev, dtype=np.float64)


def test_predict_changes_no_slot(ba):
    """twin slots, one queried many times between pushes: the same poses, released rows and save blobs"""
    st = ImuStream(ba)
    a, b = 900, 901
    st.reset([a, b])
    rng = np.random.default_rng(14)
    _feed(st, [a, b], _head())
    x = _state(rng)
    st.push([StreamRecord(a).set_state(0.02, x), StreamRecord(b).set_state(0.02, x)])
    P = _spd(rng)
    st.set_covariance([a, b], [0.02, 0.02], [P, P], NOISE)
    t = 0.06
    for k in range(30):
        st.predict([a], [np.sort(rng.uniform(0.0, t + 0.05, 5))], states=True)
        ev = []
        for _ in range(3):
            t += 0.004
            ev += [(G, t, *rng.normal(size=3)), (A, t + 0.001, 0, 0, 9.8)]
        if k % 4 == 0:
            ev.append((C, t - 0.002, 0, 0, 0))
        ev = np.array(ev)
        while len(ev):
            oa, ob = st.push([StreamRecord(a, ev), StreamRecord(b, ev)])
            assert oa["n_consumed"] == ob["n_consumed"]
            assert np.array_equal(_bits(oa["poses"]), _bits(ob["poses"]))
            assert [(f, _bits(r).tolist()) for f, r in oa["frames"]] == [(f, _bits(r).tolist()) for f, r in ob["frames"]]
            ev = ev[oa["n_consumed"]:]
        if k == 10:                                          # a new state with its drop pending, then more queries
            y = _state(rng)
            st.push([StreamRecord(a).set_state(t - 0.01, y), StreamRecord(b).set_state(t - 0.01, y)])
    ba_, bb = st.save([a, b])
    assert ba_ == bb
    pa, pb = st.predict([a, b], [[t, t + 0.1]] * 2, states=True)
    assert np.array_equal(_bits(pa["poses"]), _bits(pb["poses"]))
    assert pa["status"] == pb["status"] == NO_COVARIANCE


def test_seed_validity(ba):
    st = ImuStream(ba)
    s = 950
    st.reset([s])
    rng = np.random.default_rng(15)
    _feed(st, [s], _head())
    x, y = _state(rng), _state(rng)
    P = _spd(rng)

    def status():
        return st.predict([s], [[0.03, 0.1]])[0]["status"]

    def seed(t):
        st.set_covariance([s], [t], [P], NOISE)
        assert status() == 0
    assert status() == NO_STATE
    d = st.predict([s], [[0.03, 0.1]], states=True)[0]
    assert not d["poses"].any() and not d["states"].any() and np.isnan(d["state_cov"]).all()
    assert np.isnan(d["pose_cov"]).all()
    st.push([StreamRecord(s).set_state(0.02, x)])
    assert status() == NO_COVARIANCE
    d = st.predict([s], [[0.03]])[0]
    assert d["poses"].any() and np.isnan(d["state_cov"]).all() and np.isnan(d["pose_cov"]).all()
    seed(0.02)
    st.push([StreamRecord(s, _head(0.2, 2))])                 # KEEP: the seed holds
    assert status() == 0
    st.push([StreamRecord(s).set_state(0.02, x)])             # the same state again
    assert status() == NO_COVARIANCE
    seed(0.02)
    st.push([StreamRecord(s).set_state(0.03, y)])             # another state
    assert status() == NO_COVARIANCE
    seed(0.03)
    st.push([StreamRecord(s).clear_state()])
    assert status() == NO_STATE
    st.push([StreamRecord(s).set_state(0.03, y)])
    assert status() == NO_COVARIANCE
    seed(0.03)
    blob = st.save([s])[0]
    st.restore([s], [blob])
    assert status() == NO_COVARIANCE
    seed(0.03)
    st.reset([s])
    assert status() == NO_STATE


def test_rejections_change_no_seed_and_no_output(ba):
    st = ImuStream(ba)
    lib, h = ba.lib, ba.h
    a, b, never = 1100, 1101, 1199
    st.reset([a, b])
    rng = np.random.default_rng(16)
    _feed(st, [a, b], _head())
    st.push([StreamRecord(a).set_state(0.02, _state(rng))])
    P = _spd(rng)
    st.set_covariance([a], [0.02], [P], NOISE)
    before = st.predict([a, b], [[0.03, 0.05]] * 2, states=True)
    keep = []

    def seed(slot=a, mode=_lib.IMU_STREAM_COV_DIRECT, t=0.02, cov=P, rec=None, noise=NOISE):
        r = _lib.CImuStreamCovSeed()
        arrs = [None if v is None else np.ascontiguousarray(v, dtype=np.float64) for v in (cov, rec, noise)]
        keep.extend(arrs)
        r.slot, r.mode, r.state_time = slot, mode, t
        _lib.set_ptrs(r, cov=arrs[0], imu_record=arrs[1], noise_cov=arrs[2])
        return r

    def rejected_seed(*recs):
        arr = (_lib.CImuStreamCovSeed * len(recs))(*recs)
        assert lib.pvio_b200_batch_imu_stream_set_covariance(h, len(recs), arr) == _lib.EINVAL
        after = st.predict([a, b], [[0.03, 0.05]] * 2, states=True)
        for x, y in zip(before, after):
            assert x["status"] == y["status"]
            for k in ("poses", "states", "state_cov", "pose_cov"):
                assert np.array_equal(_bits(x[k]), _bits(y[k])), k

    Q = _spd(rng)
    asym = Q.copy()
    asym[0, 1] += 1e-9 * np.abs(Q).max()
    negd = Q.copy()
    negd[3, 3] = -1e-9
    rec = imu_oracle.record(imu_oracle.integrate(_head()[::2, [1, 2, 3, 4, 2, 3, 4]], 0.06, np.zeros(3), np.zeros(3),
                                                 *co.noise_blocks(NOISE)), np.zeros(3), np.zeros(3))
    rec_nan = rec.copy()
    rec_nan[3] = np.nan
    rejected_seed(seed(cov=Q), seed(cov=Q))                                         # a slot twice
    rejected_seed(seed(cov=Q), seed(slot=never))                                     # never reset
    rejected_seed(seed(slot=70000))                                                  # out of range
    rejected_seed(seed(cov=Q), seed(slot=b))                                         # no latest state
    rejected_seed(seed(cov=Q, t=0.021))                                              # another state time
    rejected_seed(seed(cov=Q, mode=7))                                               # unknown mode
    rejected_seed(seed(cov=None))                                                    # missing arrays
    rejected_seed(seed(cov=Q, noise=None))
    rejected_seed(seed(cov=Q, mode=_lib.IMU_STREAM_COV_FACTOR))
    q_nan = Q.copy()
    q_nan[4, 4] = np.inf
    rejected_seed(seed(cov=q_nan))                                                   # not finite
    rejected_seed(seed(cov=Q, noise=np.full(36, np.nan)))
    rejected_seed(seed(cov=Q, mode=_lib.IMU_STREAM_COV_FACTOR, rec=rec_nan))
    rejected_seed(seed(cov=asym))                                                    # not symmetric
    rejected_seed(seed(cov=negd))                                                    # a negative diagonal
    st.set_covariance([a], [0.02], [Q], NOISE, imu_records=[rec])                    # accepted: FACTOR
    assert st.predict([a], [[0.03]])[0]["status"] == 0

    def pred(slot=a, times=(0.03, 0.05), null_times=False, null_poses=False, n_times=None):
        t = np.ascontiguousarray(times, dtype=np.float64)
        o = dict(poses=np.full((4, 7), -1.0), states=np.full((4, 16), -1.0), pose_cov=np.full((4, 36), -1.0),
                 state_cov=np.full((4, 225), -1.0))
        keep.extend([t] + list(o.values()))
        r = _lib.CImuStreamPredict()
        r.slot, r.n_times, r.status = slot, len(t) if n_times is None else n_times, -3
        _lib.set_ptrs(r, times=None if null_times else t, poses=None if null_poses else o["poses"],
                      states=o["states"], pose_cov=o["pose_cov"], state_cov=o["state_cov"])
        return r, o

    def rejected_predict(*rs):
        arr = (_lib.CImuStreamPredict * len(rs))(*[r for r, _ in rs])
        assert lib.pvio_b200_batch_imu_stream_predict(h, len(rs), arr) == _lib.EINVAL
        for r, (_, o) in zip(arr, rs):
            assert r.status == -3
            for v in o.values():
                assert (v == -1).all()
    rejected_predict(pred(), pred())                                                 # a slot twice
    rejected_predict(pred(), pred(slot=never))                                       # never reset
    rejected_predict(pred(slot=-1))                                                  # out of range
    rejected_predict(pred(n_times=-1))
    rejected_predict(pred(b), pred(null_times=True))
    rejected_predict(pred(null_poses=True))
    rejected_predict(pred(times=(0.03, np.nan)))
    rejected_predict(pred(b), pred(times=(0.05, 0.03)))                              # decreasing
    r, o = pred(b, times=(0.03,))
    arr = (_lib.CImuStreamPredict * 1)(r)
    assert lib.pvio_b200_batch_imu_stream_predict(h, 1, arr) == 0 and arr[0].status == NO_STATE
    with pytest.raises(PvioB200Error):
        st.predict([a], [[0.05, 0.01]])


def test_launches_do_not_grow_with_the_batch(ba):
    st = ImuStream(ba)
    rng = np.random.default_rng(17)
    per = {}
    for n in (8, 264):
        slots = list(range(2000, 2000 + n))
        st.reset(slots)
        _feed(st, slots, _head())
        x = _state(rng)
        st.push([StreamRecord(s).set_state(0.02, x) for s in slots])
        l0 = ba.kernel_launches
        st.set_covariance(slots, [0.02] * n, [_spd(rng)] * n, NOISE)
        l1 = ba.kernel_launches
        st.predict(slots, [[0.01, 0.03, 0.05]] * n, states=True)
        l2 = ba.kernel_launches
        st.push([StreamRecord(s, _head(0.1, 3)) for s in slots])
        l3 = ba.kernel_launches
        per[n] = (l1 - l0, l2 - l1, l3 - l2)
    assert per[8] == per[264] == (1, 1, 1)
