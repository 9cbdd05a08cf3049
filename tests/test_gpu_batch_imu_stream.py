"""pvio_b200_batch_imu_stream against oracle/imu_stream_oracle.py, bit for bit: 264 sequences of mixed stream shapes
(gyroscope and accelerometer rates, equal stamps in both arrival orders, jitter, gaps, gyroscope restarts, camera
stamps behind the IMU, long chunks and one-event chunks), with a latest state injected at every release and cleared now
and then.  Every pose, n_consumed and released list is compared.  The oracle is given the device's sin / cos of the
same arguments (torch on the same GPU), the one function the two sides do not share.  Also: a batch equals each
sequence run alone, launches do not grow with the batch, and every rejection leaves the slots and outputs unchanged."""
import math

import numpy as np
import pytest

from oracle import imu_stream_oracle as so
from pvio_b200 import _lib
from pvio_b200.bundle_adjustor import BundleAdjustor, PvioB200Error
from pvio_b200.imu_stream import ImuStream, StreamRecord

pytestmark = pytest.mark.gpu
G, A, C = so.GYROSCOPE, so.ACCELEROMETER, so.CAMERA


def _events(seed):
    """one sequence's arrival-ordered events over about 1.5 s"""
    rng = np.random.default_rng(seed)
    shape = seed % 6
    t_end = 1.5
    g_dt = [0.005, 0.005, 0.0025, 0.01, 0.005, 0.001][shape]
    a_dt = g_dt if shape in (0, 1) else [0.004, 0.0075, 0.004, 0.005][shape - 2]
    jit = 0.0 if shape in (0, 1) else 2e-4
    gt = np.cumsum(np.full(int(t_end / g_dt), g_dt) + rng.uniform(0, jit, int(t_end / g_dt)))
    at = np.cumsum(np.full(int(t_end / a_dt), a_dt) + rng.uniform(0, jit, int(t_end / a_dt))) + rng.uniform(0, 3e-3)
    if shape in (0, 1):
        at = gt.copy()
    if shape == 3:                                      # a gap in the gyroscope
        gt = gt[(gt < 0.6) | (gt > 0.75)]
    cam = np.arange(0.02 + rng.uniform(0, 0.02), t_end, 0.05)
    lat = rng.uniform(0, 0.012) if shape in (2, 4) else 0.0        # camera frames arrive after newer IMU readings
    ev = []
    for t in gt:
        ev.append((t, 0 if shape != 1 else 1, (G, t, *(rng.normal(size=3) * 0.5))))
    for t in at:
        ev.append((t, 1 if shape != 1 else 0, (A, t, *(np.array([0, 0, 9.8]) + rng.normal(size=3) * 0.3))))
    for t in cam:
        ev.append((t + lat, 2, (C, t, 0.0, 0.0, 0.0)))
    ev.sort(key=lambda e: (e[0], e[1]))
    out = [e[2] for e in ev]
    if shape == 5:                                      # a gyroscope restart: readings older than the queued accelerometer
        k = len(out) // 2
        t_acc = next(e[1] for e in out[k:] if e[0] == A)
        out.insert(k, (A, t_acc + 0.004, 0.1, 0.2, 9.7))
        out = [e for e in out if not (e[0] == A and t_acc <= e[1] < t_acc + 0.004)]
    return np.array(out, dtype=np.float64)


def _state(rng, t):
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    return t, np.concatenate([q, rng.normal(size=3), rng.normal(size=3) * 0.5, rng.normal(size=3) * 0.01,
                              rng.normal(size=3) * 0.05])


class _Seq:
    def __init__(self, seed):
        self.ev, self.pos, self.seed = _events(seed), 0, seed
        self.rng = np.random.default_rng(1000 + seed)
        self.pending = None                              # (op, state) for the next push
        self.calls = []                                  # (events, op, state) of every push, for the oracle

    def record(self, slot):
        lo = self.pos
        n = 1 if self.rng.random() < 0.2 else int(self.rng.integers(1, 40))
        r = StreamRecord(slot, self.ev[lo:lo + n])
        op = self.pending
        if op is not None and op[0] == "set":
            r.set_state(*op[1])
        elif op is not None:
            r.clear_state()
        self.calls.append((self.ev[lo:lo + n], op))
        self.pending = None
        return r

    def took(self, out):
        self.pos += out["n_consumed"]
        if out["frames"]:
            t = out["frames"][-1][0]
            self.pending = ("clear", None) if self.rng.random() < 0.05 else ("set", _state(self.rng, t))

    @property
    def done(self):
        return self.pos >= len(self.ev)


def _drive(stream, seqs, slots):
    results = [[] for _ in seqs]
    while True:
        live = [i for i, s in enumerate(seqs) if not s.done]
        if not live:
            return results
        outs = stream.push([seqs[i].record(slots[i]) for i in live])
        for i, o in zip(live, outs):
            seqs[i].took(o)
            results[i].append(o)


def _oracle(seq, sincos):
    st = so.Stream(sincos=sincos)
    res = []
    for ev, op in seq.calls:
        poses, n, rel = st.push(ev, state=op[1] if op and op[0] == "set" else None, clear=bool(op and op[0] == "clear"))
        res.append((np.array(poses).reshape(-1, 7), n, rel))
    return res


def _device_sincos(seqs):
    """the device's sin / cos of every argument the oracle needs (both sides compute the arguments identically)"""
    import torch
    args = set()

    def record(x):
        args.add(x)
        return math.sin(x), math.cos(x)
    for s in seqs:
        _oracle(s, record)
    xs = sorted(args)
    x = torch.tensor(xs, dtype=torch.float64, device="cuda")
    table = dict(zip(xs, zip(torch.sin(x).cpu().tolist(), torch.cos(x).cpu().tolist())))

    def sincos(v):
        if v not in table:
            y = torch.tensor([v], dtype=torch.float64, device="cuda")
            table[v] = (torch.sin(y).item(), torch.cos(y).item())
        return table[v]
    return sincos


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _same(dev, ref):
    assert len(dev) == len(ref)
    for o, (poses, n, rel) in zip(dev, ref):
        assert o["n_consumed"] == n
        assert np.array_equal(_bits(o["poses"]), _bits(poses))
        assert len(o["frames"]) == len(rel)
        for (t, rows), (rt, rrows) in zip(o["frames"], rel):
            assert t == rt
            assert np.array_equal(_bits(rows.reshape(-1, 7)), _bits(np.array(rrows).reshape(-1, 7)))


@pytest.fixture(scope="module")
def ba():
    b = BundleAdjustor(max_windows=1, max_frames=8, max_landmarks=64, max_obs=256)
    yield b
    b.close()


def test_264_mixed_sequences_bit_equal_to_the_oracle_and_each_alone(ba):
    st = ImuStream(ba)
    n = 264
    seqs = [_Seq(s) for s in range(n)]
    slots = list(range(5, 5 + n))
    rng = np.random.default_rng(7)
    q_ob = np.array([0.0, 0.0, 0.0, 1.0])
    st.reset(slots, q_ob, np.zeros(3))
    res = _drive(st, seqs, slots)
    sincos = _device_sincos(seqs)
    released = 0
    for s, r in zip(seqs, res):
        _same(r, _oracle(s, sincos))
        released += sum(len(o["frames"]) for o in r)
    assert released > 20 * n
    # alone: the same calls, one sequence per call, in other slots with an output extrinsic; and the batch slots stay
    q_x = rng.normal(size=4)
    q_x /= np.linalg.norm(q_x)
    p_x = np.array([0.1, -0.2, 0.05])
    for k in range(0, n, 33):
        s = seqs[k]
        st.reset([400], q_x, p_x)
        alone = []
        for ev, op in s.calls:
            r = StreamRecord(400, ev)
            if op and op[0] == "set":
                r.set_state(*op[1])
            elif op:
                r.clear_state()
            alone.append(st.push([r])[0])
        o2 = so.Stream(q_x, p_x, sincos=sincos)
        ref = []
        for ev, op in s.calls:
            poses, nn, rel = o2.push(ev, state=op[1] if op and op[0] == "set" else None,
                                     clear=bool(op and op[0] == "clear"))
            ref.append((np.array(poses).reshape(-1, 7), nn, rel))
        _same(alone, ref)
    # the batch slots are untouched by the runs in slot 400: one more event continues each oracle stream
    probe = [StreamRecord(slots[i], [(C, 10.0, 0, 0, 0)]) for i in range(0, n, 11)]
    outs = st.push(probe)
    for i, o in zip(range(0, n, 11), outs):
        o3 = so.Stream(sincos=sincos)
        for ev, op in seqs[i].calls:
            o3.push(ev, state=op[1] if op and op[0] == "set" else None, clear=bool(op and op[0] == "clear"))
        p, _, _ = o3.push([(C, 10.0, 0, 0, 0)])
        assert np.array_equal(_bits(o["poses"]), _bits(np.array(p))), i


def test_batch_equals_each_sequence_alone_bit_for_bit(ba):
    st = ImuStream(ba)
    seqs = [_Seq(s) for s in range(24)]
    slots = list(range(24))
    st.reset(slots)
    res = _drive(st, seqs, slots)
    for k in (0, 5, 11, 23):
        st.reset([500])
        alone = []
        for ev, op in seqs[k].calls:
            r = StreamRecord(500, ev)
            if op and op[0] == "set":
                r.set_state(*op[1])
            elif op:
                r.clear_state()
            alone.append(st.push([r])[0])
        assert len(alone) == len(res[k])
        for a, b in zip(alone, res[k]):
            assert a["n_consumed"] == b["n_consumed"]
            assert np.array_equal(_bits(a["poses"]), _bits(b["poses"]))
            assert [(t, _bits(r).tolist()) for t, r in a["frames"]] == [(t, _bits(r).tolist()) for t, r in b["frames"]]


def test_launches_do_not_grow_with_the_batch(ba):
    st = ImuStream(ba)
    per_call = {}
    for n in (8, 264):
        slots = list(range(1000, 1000 + n))
        st.reset(slots)
        ev = []
        for k in range(10):
            t = 0.005 * k
            ev += [(G, t, 0.1, 0.2, 0.3), (A, t, 0.0, 0.0, 9.8)]
        ev.append((C, 0.047, 0, 0, 0))
        st.push([StreamRecord(s, ev) for s in slots])            # grows the queues
        ev2 = [(e[0], e[1] + 0.05, *e[2:]) for e in ev]
        l0 = ba.kernel_launches
        st.push([StreamRecord(s, ev2) for s in slots])
        per_call[n] = ba.kernel_launches - l0
    assert per_call[8] == per_call[264] == 1


def test_rejections_change_no_slot_and_no_output(ba):
    st = ImuStream(ba)
    lib, h = ba.lib, ba.h
    a_slot, b_slot = 2000, 2001
    st.reset([a_slot, b_slot])
    head = [(G, 0.0, 0.1, 0.2, 0.3), (A, 0.0, 0, 0, 9.8), (C, 0.02, 0, 0, 0), (G, 0.01, 0.1, 0.2, 0.3),
            (A, 0.01, 0, 0, 9.8), (G, 0.03, 0.2, 0.1, 0.0), (A, 0.03, 0.1, 0, 9.7)]
    for s in (a_slot, b_slot):
        ev = head
        while ev:
            o = st.push([StreamRecord(s, ev)])[0]
            ev = ev[o["n_consumed"]:]
    st.push([StreamRecord(a_slot).set_state(*_state(np.random.default_rng(1), 0.02)),
             StreamRecord(b_slot).set_state(*_state(np.random.default_rng(1), 0.02))])

    def raw(slot, events, state_op=_lib.IMU_STREAM_KEEP, state=None, state_time=0.0, max_frames=8, max_rows=64,
            rows=True):
        ev = np.ascontiguousarray(np.asarray(events, dtype=np.float64).reshape(-1, 5))
        r = _lib.CImuStreamRecord()
        bufs = dict(poses=np.full((max(len(ev), 1), 7), -1.0), frame_t=np.full(max(max_frames, 1), -1.0),
                    frame_rows=np.full(max(max_frames, 1), -1, np.int32), rows=np.full((max(max_rows, 1), 7), -1.0))
        r.slot, r.n_events, r.state_op, r.state_time = slot, len(ev), state_op, state_time
        r.max_frames, r.max_rows = max_frames, max_rows
        r.n_consumed = r.n_frames = -3
        _lib.set_ptrs(r, events=ev if len(ev) else None, state=state, poses=bufs["poses"], frame_t=bufs["frame_t"],
                      frame_rows=bufs["frame_rows"], rows=bufs["rows"] if rows else None)
        return r, bufs, ev

    def rejected(*recs):
        arr = (_lib.CImuStreamRecord * len(recs))(*[r for r, _, _ in recs])
        assert lib.pvio_b200_batch_imu_stream(h, len(recs), arr) == _lib.EINVAL
        for (_, bufs, _), r in zip(recs, arr):
            assert r.n_consumed == -3 and r.n_frames == -3
            for k, v in bufs.items():
                assert (v == -1).all(), k

    ok = [(G, 0.04, 0.1, 0.1, 0.1)]
    rejected(raw(a_slot, ok), raw(a_slot, ok))                                     # a slot twice
    rejected(raw(a_slot, ok), raw(3000, ok))                                       # never reset
    rejected(raw(a_slot, ok), raw(70000, ok))                                      # out of range
    rejected(raw(a_slot, [(7, 0.04, 0, 0, 0)]))                                    # unknown kind
    rejected(raw(a_slot, [(0.5, 0.04, 0, 0, 0)]))
    rejected(raw(a_slot, [(G, 0.04, np.nan, 0, 0)]))                               # not finite
    rejected(raw(a_slot, [(A, 0.04, 0, np.inf, 0)]))
    rejected(raw(a_slot, ok + [(G, 0.035, 0, 0, 0)]))                              # a gyroscope time decreases
    rejected(raw(a_slot, [(A, 0.02, 0, 0, 9.8)]))                                  # an accelerometer time decreases
    rejected(raw(a_slot, ok, state_op=5))                                          # unknown state_op
    rejected(raw(a_slot, ok, state_op=_lib.IMU_STREAM_SET))                        # SET without a state
    rejected(raw(a_slot, ok, state_op=_lib.IMU_STREAM_SET, state=np.full(16, np.nan)))
    rejected(raw(a_slot, [(A, 0.05, 0, 0, 9.8), (G, 0.06, 0, 0, 0), (C, 0.055, 0, 0, 0)], max_rows=0))  # room
    rejected(raw(a_slot, [(C, 0.05 + 0.001 * k, 0, 0, 0) for k in range(3)], max_frames=1))
    big = [(G, 0.04 + 1e-6 * k, 0, 0, 0) for k in range(_lib.IMU_STREAM_MAX_QUEUE + 1)]
    rejected(raw(a_slot, big, max_rows=8))                                         # a queue past the limit
    # a state older than a frame released while the slot had none
    c_slot = 2002
    st.reset([c_slot])
    ev = head
    while ev:
        ev = ev[st.push([StreamRecord(c_slot, ev)])[0]["n_consumed"]:]
    rejected(raw(c_slot, ok, state_op=_lib.IMU_STREAM_SET, state=_state(np.random.default_rng(2), 0.0)[1],
                 state_time=0.015))
    # size query: writes the needs only
    r, bufs, _ = raw(a_slot, [(A, 0.05, 0, 0, 9.8), (G, 0.06, 0, 0, 0)], rows=False)
    arr = (_lib.CImuStreamRecord * 1)(r)
    assert lib.pvio_b200_batch_imu_stream(h, 1, arr) == 0
    assert arr[0].need_rows >= 2 and arr[0].n_consumed == -3 and (bufs["poses"] == -1).all()
    # the twins still agree, event by event
    rng = np.random.default_rng(4)
    t = 0.04
    for _ in range(40):
        ev = []
        for _ in range(int(rng.integers(1, 6))):
            t += 0.004
            ev += [(G, t, *rng.normal(size=3)), (A, t + 0.001, 0, 0, 9.8)]
        if rng.random() < 0.4:
            ev.append((C, t - 0.002, 0, 0, 0))
        while ev:
            oa, ob = st.push([StreamRecord(a_slot, ev), StreamRecord(b_slot, ev)])
            assert oa["n_consumed"] == ob["n_consumed"]
            assert np.array_equal(_bits(oa["poses"]), _bits(ob["poses"]))
            assert len(oa["frames"]) == len(ob["frames"])
            for (ta, ra), (tb, rb) in zip(oa["frames"], ob["frames"]):
                assert ta == tb and np.array_equal(_bits(ra), _bits(rb))
            ev = ev[oa["n_consumed"]:]
    with pytest.raises(PvioB200Error):
        st.push([StreamRecord(a_slot, [(G, 0.0, 0, 0, 0)])])


def test_a_state_drops_samples_only_when_a_pose_reads_it(ba):
    """a state set by a record without events, then replaced by an older one before any pose: the older state still
    propagates over the samples between the two times, as predict_pose pops only when it runs"""
    st = ImuStream(ba)
    slot = 2100
    st.reset([slot])
    ev = []
    for k in range(40):
        t = 0.005 * k
        ev += [(G, t, 0.3, -0.2, 0.1 + t), (A, t, 0.1, 0.2, 9.8 - t)]
    ev = np.array(ev)
    pos = 0
    calls = []
    while pos < len(ev):                                 # no camera stamp: everything is consumed, nothing released
        o = st.push([StreamRecord(slot, ev[pos:pos + 25])])[0]
        calls.append((ev[pos:pos + 25], None))
        pos += o["n_consumed"]
    s_late, s_early = _state(np.random.default_rng(5), 0.15), _state(np.random.default_rng(6), 0.05)
    st.push([StreamRecord(slot).set_state(*s_late)])
    tail = [(C, 0.19, 0, 0, 0), (C, 0.12, 0, 0, 0)]
    out = st.push([StreamRecord(slot, tail).set_state(*s_early)])[0]
    seq = _Seq(0)
    seq.calls = calls + [(np.zeros((0, 5)), ("set", s_late)), (np.array(tail, dtype=np.float64), ("set", s_early))]
    ref = _oracle(seq, _device_sincos([seq]))
    assert out["n_consumed"] == 2
    assert np.array_equal(_bits(out["poses"]), _bits(ref[-1][0]))
    assert ref[-1][0][0, 4:].any()
