"""pvio_b200_batch_imu_stream_save / pvio_b200_batch_imu_stream_restore: stream slots saved to host memory at awkward
moments (before the first camera stamp, camera stamps ahead of the IMU, unreleased samples on the front frame, no state
after releases that dropped kept samples, a pending drop from a zero-event SET, a cleared state, a queued gyroscope
backlog) and restored into other slots of the same handle and into a fresh, smaller handle.  Every copy must then
continue bit for bit as its source does, and the source as oracle/imu_stream_oracle.py.  Also: forks and a rollback,
every rejection leaving every slot as it was, one launch per call whatever n is, and a running closed-loop sequence
(stream slot, window slot and tracker slot) moved to a second handle."""
import numpy as np
import pytest

from oracle import imu_stream_oracle as so
from pvio_b200 import _lib
from pvio_b200.batch_window import BatchWindows, Camera, Edit
from pvio_b200.bundle_adjustor import BundleAdjustor, PvioB200Error
from pvio_b200.imu_stream import ImuStream, StreamRecord
from test_gpu_batch_imu_stream import _Seq, _device_sincos, _drive, _events, _oracle, _same
from test_gpu_batch_window_mirror import SEQ_TOL
from test_gpu_batch_window_track_camera import CAP, KD, Seq, _start, _state16
from test_gpu_imu_stream_closed_loop import _events as _loop_events

pytestmark = pytest.mark.gpu
G, A, C = so.GYROSCOPE, so.ACCELEROMETER, so.CAMERA
CUTS = (0, 2, 5, 12, 30, 70)                 # drive rounds after which every stream slot is saved
# the blob head (csrc/imu_stream.cu: StreamSnapHead): name -> (byte offset, dtype)
HEAD = dict(magic=(0, "<u4"), version=(4, "<u4"), size=(8, "<i8"), n0=(16, "<i4"), n1=(20, "<i4"), n2=(24, "<i4"),
            n3=(28, "<i4"), n4=(32, "<i4"), seen_g=(36, "<i4"), seen_a=(40, "<i4"), dropped=(44, "<i4"),
            last_g=(48, "<f8"), last_a=(56, "<f8"), t_drop=(64, "<f8"), q_ob=(72, "<f8"), p_ob=(104, "<f8"),
            state_t=(128, "<f8"), state=(136, "<f8"), prev_t=(264, "<f8"), prev_row=(272, "<f8"),
            has_state=(320, "<i4"), drop_pending=(324, "<i4"), has_prev=(328, "<i4"), prev_nonempty=(332, "<i4"),
            nfront=(336, "<i4"), pad=(340, "<i4"))
HEAD_BYTES = 344
WIDTH = (4, 4, 7, 1, 7)                      # g, a, s, f, k rows


def _get(blob, k):
    o, t = HEAD[k]
    return np.frombuffer(blob, dtype=t, count=1, offset=o)[0].item()


def _poke(blob, off, dtype, v):
    out = bytearray(blob)
    out[off:off + np.dtype(dtype).itemsize] = np.array([v], dtype=dtype).tobytes()
    return bytes(out)


def _put(blob, k, v):
    return _poke(blob, HEAD[k][0], HEAD[k][1], v)


def _section(blob, q):
    """byte offset of queue q's rows"""
    return HEAD_BYTES + 8 * sum(WIDTH[j] * _get(blob, f"n{j}") for j in range(q))


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _equal_outs(a, b):
    assert a["n_consumed"] == b["n_consumed"]
    assert np.array_equal(_bits(a["poses"]), _bits(b["poses"]))
    assert len(a["frames"]) == len(b["frames"])
    for (ta, ra), (tb, rb) in zip(a["frames"], b["frames"]):
        assert ta == tb and np.array_equal(_bits(ra), _bits(rb))


def _clone(r, slot):
    c = StreamRecord(slot, r.events)
    c.state_op, c.state_time, c.state = r.state_op, r.state_time, r.state
    return c


def _sizes(st, slots):
    recs = (_lib.CImuStreamSnapshot * len(slots))()
    for r, s in zip(recs, slots):
        r.slot = s
    n0 = st.ba.kernel_launches
    assert st.lib.pvio_b200_batch_imu_stream_save(st.h, len(slots), recs) == 0
    assert st.ba.kernel_launches == n0                   # a size query does no device work
    return [r.size for r in recs]


def _cut_events(seed):
    """_events, and every eleventh sequence with no camera stamp before 0.4 s: a backlog of unreleased samples"""
    ev = _events(seed)
    if seed % 11 == 0:
        ev = ev[(ev[:, 0] != C) | (ev[:, 1] >= 0.4)]
    return ev


@pytest.fixture(scope="module")
def ba():
    b = BundleAdjustor(max_windows=1, max_frames=8, max_landmarks=64, max_obs=256)
    yield b
    b.close()


def test_round_trip_at_awkward_moments(ba):
    st = ImuStream(ba)
    n = 264
    seqs = [_Seq(s) for s in range(n)]
    for s in seqs:
        s.ev = _cut_events(s.seed)
        s.cleared = False
    slots = list(range(5, 5 + n))
    st.reset(slots)
    fresh = BundleAdjustor(max_windows=1, max_frames=8, max_landmarks=64, max_obs=256)
    try:
        sf = ImuStream(fresh)
        sf.reset([0])                                    # the fewest stream slots and the smallest queues
        copies = []                                      # (stream, slot of each sequence)
        res = [[] for _ in seqs]
        seen = dict(no_camera=0, pending=0, nfront=0, dropped=0, drop_pending=0, cleared=0, gyro2=0, backlog=0)

        def push(idx, recs):
            outs = st.push(recs)
            for i, o in zip(idx, outs):
                res[i].append(o)
            for cs, cslots in copies:
                for o, c in zip(outs, cs.push([_clone(r, cslots[i]) for i, r in zip(idx, recs)])):
                    _equal_outs(o, c)
            return outs

        for rnd in range(10 ** 6):
            live = [i for i, s in enumerate(seqs) if not s.done]
            if not live:
                break
            recs = [seqs[i].record(slots[i]) for i in live]
            for i, r in zip(live, recs):
                if r.state_op == _lib.IMU_STREAM_CLEAR:
                    seqs[i].cleared = True
                elif r.state_op == _lib.IMU_STREAM_SET:
                    seqs[i].cleared = False
            for i, o in zip(live, push(live, recs)):
                seqs[i].took(o)
            if rnd not in CUTS:
                continue
            # even sequences with a state to feed back take it in a zero-event record: a pending drop
            zero = [i for i in live if i % 2 == 0 and seqs[i].pending and seqs[i].pending[0] == "set"]
            zrecs = []
            for i in zero:
                zrecs.append(StreamRecord(slots[i]).set_state(*seqs[i].pending[1]))
                seqs[i].calls.append((np.zeros((0, 5)), seqs[i].pending))
                seqs[i].pending, seqs[i].cleared = None, False
            if zero:
                push(zero, zrecs)
            blobs = st.save(slots)
            assert _sizes(st, slots) == [len(b) for b in blobs]
            for i, (s, b) in enumerate(zip(seqs, blobs)):
                cnt = [_get(b, f"n{q}") for q in range(5)]
                seen["no_camera"] += (not (s.ev[:s.pos, 0] == C).any()) and sum(cnt) > 0
                seen["pending"] += cnt[3] > 0
                seen["nfront"] += _get(b, "nfront") > 0
                seen["dropped"] += _get(b, "has_state") == 0 and _get(b, "dropped") == 1
                seen["drop_pending"] += _get(b, "drop_pending")
                seen["cleared"] += s.cleared and _get(b, "has_state") == 0
                seen["gyro2"] += cnt[0] >= 2
                seen["backlog"] += max(cnt) > 16
            c = len(copies) // 2
            same = [2000 + 300 * c + i for i in range(n)]
            other = [100 + 300 * c + i for i in range(n)]
            st.restore(same, blobs)
            sf.restore(other, blobs)                     # grows the fresh handle's slots and queues
            assert st.save(same) == blobs and sf.save(other) == blobs
            copies += [(st, same), (sf, other)]
        assert len(copies) == 2 * len(CUTS)
        print("cuts:", seen)
        assert all(v > 0 for v in seen.values()), seen
        final = st.save(slots)
        for cs, cslots in copies:
            assert cs.save(cslots) == final
        sincos = _device_sincos(seqs)
        for s, r in zip(seqs, res):
            _same(r, _oracle(s, sincos))
    finally:
        fresh.close()


def test_fork_and_rollback(ba):
    st = ImuStream(ba)
    seqs = [_Seq(s) for s in (2, 3, 4, 5)]
    slots = [3000 + j for j in range(len(seqs))]
    st.reset(slots)
    for _ in range(8):                                   # part of the way
        live = [i for i, s in enumerate(seqs) if not s.done]
        for i, o in zip(live, st.push([seqs[i].record(slots[i]) for i in live])):
            seqs[i].took(o)
    src = slots[1]
    s = seqs[1]
    blob = st.save([src])[0]
    mark, pos0 = len(s.calls), s.pos
    first = _drive(st, [s], [src])[0]                    # the first pass from the save
    replay = s.calls[mark:]

    def records(slot, calls, scale=1.0):
        out = []
        for ev, op in calls:
            ev = np.array(ev)
            ev[:, 2:] *= scale
            r = StreamRecord(slot, ev)
            if op and op[0] == "set":
                r.set_state(*op[1])
            elif op:
                r.clear_state()
            out.append(r)
        return out

    def run(slot, calls, scale=1.0):
        return [st.push([r])[0] for r in records(slot, calls, scale)]      # the first pass's records again

    forks = [3100, 3101, 3102]
    st.restore(forks, [blob] * 3)                        # one blob into three slots: a fork
    assert st.save(forks) == [blob] * 3
    same = run(forks[0], replay)
    louder = run(forks[1], replay, 1.5)
    for a, b in zip(same, first):
        _equal_outs(a, b)
    # the third continues with other states and chunks: the lockstep rule still consumes every event
    rng = np.random.default_rng(11)
    ev = s.ev[pos0:]
    pos, other = 0, []
    while pos < len(ev):
        r = StreamRecord(forks[2], ev[pos:pos + int(rng.integers(1, 9))])
        if other and other[-1]["frames"]:
            r.set_state(other[-1]["frames"][-1][0], np.r_[[0, 0, 0, 1.0], rng.normal(size=12) * 0.1])
        other.append(st.push([r])[0])
        pos += other[-1]["n_consumed"]
    differ = lambda x, y: any(not np.array_equal(_bits(a["poses"]), _bits(b["poses"])) for a, b in zip(x, y))  # noqa: E731
    assert differ(louder, first) and np.concatenate([o["poses"] for o in other]).any()
    assert st.save([forks[0]]) == st.save([src])
    # rollback: the blob back into its source slot, the same records again
    st.restore([src], [blob])
    again = run(src, replay)
    assert len(again) == len(first)
    for a, b in zip(again, first):
        _equal_outs(a, b)


def _state(rng, t):
    q = rng.normal(size=4)
    return t, np.r_[q / np.linalg.norm(q), rng.normal(size=3), rng.normal(size=3) * 0.5, rng.normal(size=6) * 0.01]


def _fill(st, slot, accel_tail=False):
    """a slot with a state, a previous frame, two pending camera stamps, unreleased samples given to the front frame,
    kept samples, and gyroscope readings queued past the last accelerometer reading (accel_tail: accelerometer
    readings queued ahead of the gyroscope instead; the two queues never both hold two rows)"""
    ev = []
    for k in range(11):                                  # gyroscope at 1 kHz, accelerometer at 200 Hz
        ev += [(G, 0.005 * k + 0.001 * j, 0.1 * j, 0.2, -0.1) for j in range(5)] + [(A, 0.005 * k + 0.0045, 0.1, 0, 9.8)]
    ev.insert(20, (C, 0.02, 0, 0, 0))
    ev += [(C, 0.07, 0, 0, 0), (C, 0.08, 0, 0, 0), (G, 0.055, 0.3, 0.2, -0.1), (G, 0.056, 0.3, 0.2, -0.1)]
    if accel_tail:
        ev += [(A, 0.058, 0.1, 0, 9.8), (A, 0.06, 0.1, 0, 9.7)]
    ev = np.array(ev, dtype=np.float64)
    pos, state = 0, None
    while pos < len(ev):
        r = StreamRecord(slot, ev[pos:])
        if state:
            r.set_state(*state)
            state = None
        o = st.push([r])[0]
        pos += o["n_consumed"]
        if o["frames"]:
            state = _state(np.random.default_rng(3), o["frames"][-1][0])


def test_rejections_change_nothing(ba):
    st = ImuStream(ba)
    lib, h = ba.lib, ba.h
    a_slot, b_slot, tgt, d_slot = 4000, 4001, 4002, 4003
    slots = [a_slot, b_slot, tgt, d_slot]
    st.reset(slots)
    for s in slots:
        _fill(st, s, s == d_slot)
    blob, blob_a = st.save([a_slot, d_slot])
    cnt, cnt_a = [_get(blob, f"n{q}") for q in range(5)], [_get(blob_a, f"n{q}") for q in range(5)]
    assert cnt[0] >= 2 and min(cnt[2:]) >= 2 and cnt_a[1] >= 2, (cnt, cnt_a)
    assert _get(blob, "has_state") == 1 and _get(blob, "has_prev") == 1 and _get(blob, "prev_nonempty") == 1
    assert _get(blob, "dropped") == 1 and _get(blob, "nfront") >= 1
    before = st.save(slots)
    assert before[1] == before[2] == blob

    def restore(blobs, slots_):
        recs = (_lib.CImuStreamSnapshot * len(blobs))()
        arrs = [np.frombuffer(x, dtype=np.uint8) for x in blobs]
        for r, x, s in zip(recs, arrs, slots_):
            r.slot, r.data, r.capacity = s, _lib.ptr(x) if len(x) else None, len(x)
        return lib.pvio_b200_batch_imu_stream_restore(h, len(blobs), recs)

    def rejected(blobs, slots_=(tgt,)):
        assert restore(blobs, slots_) == _lib.EINVAL
        assert st.save(slots) == before

    def accepted(b):                                     # restored into tgt, then tgt put back
        assert restore([b], [tgt]) == 0
        assert restore([blob], [tgt]) == 0
        assert st.save(slots) == before

    accepted(blob)
    rejected([_put(blob, "magic", 7)])
    rejected([_put(blob, "version", 2)])
    rejected([_put(blob, "size", len(blob) + 8)])        # not the byte count
    rejected([blob[:-8]])
    rejected([blob + bytes(8)])
    rejected([_put(blob, "size", len(blob) + 8) + bytes(8)])            # the byte count, not the counts' size
    rejected([blob[:HEAD_BYTES - 8]])
    rejected([b""])
    for q in range(5):
        rejected([_put(blob, f"n{q}", cnt[q] + 1)])
        rejected([_put(blob, f"n{q}", -1)])
    # a count above the limit with a size that matches it (pending camera stamps have no order to break)
    big = _lib.IMU_STREAM_MAX_QUEUE + 1
    o3 = _section(blob, 3) + 8 * cnt[3]
    grown = _put(_put(blob, "n3", big), "size", len(blob) + 8 * (big - cnt[3]))
    rejected([grown[:o3] + bytes(8 * (big - cnt[3])) + grown[o3:]])
    rejected([_put(blob, "nfront", cnt[2] + 1)])
    rejected([_put(blob, "nfront", -1)])
    for k in ("seen_g", "seen_a", "dropped", "has_state", "drop_pending", "has_prev", "prev_nonempty"):
        rejected([_put(blob, k, 2)])
        rejected([_put(blob, k, -1)])
    rejected([_put(blob, "pad", 1)])
    rejected([_put(_put(blob, "has_state", 0), "drop_pending", 1)])     # a pending drop without a state
    rejected([_put(_put(blob, "has_prev", 0), "prev_nonempty", 1)])
    older = _put(blob, "t_drop", _get(blob, "state_t") + 1e-3)
    rejected([older])                                    # a state older than a frame released without one
    accepted(_put(_put(older, "has_state", 0), "drop_pending", 0))      # without the state it is accepted
    for k in ("last_g", "last_a", "t_drop", "q_ob", "p_ob", "state_t", "state", "prev_t", "prev_row"):
        rejected([_poke(blob, HEAD[k][0], "<f8", np.nan)])
        rejected([_poke(blob, HEAD[k][0], "<f8", -np.inf)])
    for q in range(5):                                   # a queue value that is not finite, a time that decreases
        b = blob_a if q == 1 else blob
        o = _section(b, q)
        rejected([_poke(b, o + 8 * (WIDTH[q] * _get(b, f"n{q}") - 1), "<f8", np.inf)])
        t0 = np.frombuffer(b, "<f8", count=1, offset=o)[0]
        if q != 3:
            rejected([_poke(b, o + 8 * WIDTH[q], "<f8", t0 - 1e-3)])
        else:                                            # pending camera stamps: no order check
            accepted(_poke(b, o + 8, "<f8", t0 - 1e-3))
    g_last = np.frombuffer(blob, "<f8", count=1, offset=_section(blob, 0) + 8 * 4 * (cnt[0] - 1))[0]
    a_last = np.frombuffer(blob_a, "<f8", count=1, offset=_section(blob_a, 1) + 8 * 4 * (cnt_a[1] - 1))[0]
    rejected([_put(blob, "last_g", g_last - 1e-4)])      # a queued reading newer than its stream's last
    rejected([_put(blob_a, "last_a", a_last - 1e-4)])
    rejected([_put(blob, "seen_g", 0)])                  # a non-empty queue of a stream never seen
    rejected([_put(blob_a, "seen_a", 0)])
    # a window blob
    bw = BatchWindows(ba)
    ws = Seq(0, 0, 0, 3, 1700)
    bw.reset(0, ws.run.w)
    bw.edit([Edit(0).frame(_state16(ws.run, 0))])
    rejected([bw.save([0])[0]])
    # slots out of range or named twice, and one bad record among good ones
    rejected([blob], (-1,))
    rejected([blob], (65536,))
    rejected([blob, blob], (tgt, tgt))
    rejected([blob, _put(blob, "magic", 7)], (tgt, 4004))
    # capacity one byte short of the blob, or one past it
    x = np.frombuffer(blob + bytes(1), dtype=np.uint8)
    for cap in (len(blob) - 1, len(blob) + 1):
        recs = (_lib.CImuStreamSnapshot * 1)()
        recs[0].slot, recs[0].data, recs[0].capacity = tgt, _lib.ptr(x), cap
        assert lib.pvio_b200_batch_imu_stream_restore(h, 1, recs) == _lib.EINVAL
        assert st.save(slots) == before
    # save: never reset, out of range, named twice, capacity below the size; none writes a buffer or a size
    size = _sizes(st, [a_slot])[0]
    for s_, cap in (([4999], size), ([-1], size), ([65536], size), ([a_slot, a_slot], size), ([a_slot], size - 1)):
        bufs = [np.full(size, 0xAB, dtype=np.uint8) for _ in s_]
        recs = (_lib.CImuStreamSnapshot * len(s_))()
        for r, s, b in zip(recs, s_, bufs):
            r.slot, r.data, r.capacity, r.size = s, _lib.ptr(b), cap, -5
        assert lib.pvio_b200_batch_imu_stream_save(h, len(s_), recs) == _lib.EINVAL
        assert all(r.size == -5 for r in recs) and all((b == 0xAB).all() for b in bufs)
    with pytest.raises(PvioB200Error):
        st.restore([tgt], [blob[:-8]])
    assert st.save(slots) == before
    # the twins a and b still agree, event by event, with a SET now and then
    rng = np.random.default_rng(4)
    t = 0.06
    for _ in range(30):
        ev = []
        for _ in range(int(rng.integers(1, 6))):
            t += 0.004
            ev += [(G, t, *rng.normal(size=3)), (A, t + 0.001, 0, 0, 9.8)]
        if rng.random() < 0.4:
            ev.append((C, t - 0.002, 0, 0, 0))
        while ev:
            ra, rb = StreamRecord(a_slot, ev), StreamRecord(b_slot, ev)
            if rng.random() < 0.3:
                x = _state(rng, t)
                ra.set_state(*x)
                rb.set_state(*x)
            oa, ob = st.push([ra, rb])
            _equal_outs(oa, ob)
            ev = ev[oa["n_consumed"]:]
    assert st.save([a_slot]) == st.save([b_slot])


def test_launches_do_not_depend_on_n(ba):
    st = ImuStream(ba)
    counts = []
    for n in (8, 264):
        slots = list(range(5000, 5000 + n))
        st.reset(slots)
        for s in slots[::37]:
            _fill(st, s)
        ev = [(G, 0.001 * k, 0.1, 0.2, 0.3) for k in range(3)] + [(A, 0.0015, 0, 0, 9.8), (C, 0.01, 0, 0, 0)]
        st.push([StreamRecord(s, ev) for s in slots if s not in slots[::37]])
        _sizes(st, slots)                                # no launch (checked there)
        n0 = ba.kernel_launches
        blobs = st.save(slots)
        n1 = ba.kernel_launches
        st.restore(slots, blobs)                         # the slots and their queues are already large enough
        counts.append((n1 - n0, ba.kernel_launches - n1))
        assert st.save(slots) == blobs
    assert counts == [(1, 1), (1, 1)], counts


FRAMES, MOVE = 21, 10


def _base():
    torch = pytest.importorskip("torch")
    return (torch.cuda.get_device_properties(0).multi_processor_count + 1) // 2


def _loop_handle(base):
    return BundleAdjustor(max_windows=base + 16, max_frames=9, max_landmarks=4096, max_obs=16384)


def _same_frame(x, y, exact):
    """two track_camera outputs of the same frame: integers and keypoints bit for bit, states bit for bit (exact) or
    within the repository's bar"""
    assert x["n_keypoints"] == y["n_keypoints"]
    assert np.array_equal(_bits(x["keypoints"]), _bits(y["keypoints"]))
    for key in ("prev_index", "kp_track", "counts", "feature_counts", "info"):
        assert np.array_equal(x[key], y[key]), key
    for key in ("keyframe", "n_parallax", "skipped_frames"):
        assert x[key] == y[key], key
    for key in ("state", "predicted", "imu_record"):
        if exact:
            assert np.array_equal(_bits(x[key]), _bits(y[key])), key
        else:
            assert np.abs(x[key] - y[key]).max() <= SEQ_TOL * max(1.0, np.abs(x[key]).max()), key


def test_move_a_running_sequence_to_another_handle():
    """the closed loop of test_gpu_imu_stream_closed_loop on one handle to frame MOVE; there, after a keyframe solve and
    drop, the state goes into the stream slot with a zero-event SET and the window, tracker and stream slots move to a
    second handle of the same shape; both copies then run to frame FRAMES on the same events"""
    base = _base()
    h1, h2 = _loop_handle(base), _loop_handle(base)
    try:
        bw1, st1, bw2, st2 = BatchWindows(h1), ImuStream(h1), BatchWindows(h2), ImuStream(h2)
        seqs = [Seq(j, base + j, base + 8 + j, FRAMES + 3, 1700 + j) for j in range(8)]
        _start(bw1, seqs)
        for s in seqs:
            s.events, s.state = _loop_events(s.run), None
            s.truth_t = [0.0] + [f[1] for f in s.run.truth.imu_factors]
            s.pos = {1: 0, 2: 0}
        st1.reset([s.j for s in seqs])
        where = {1: (bw1, st1), 2: (bw2, st2)}
        states = {1: {}, 2: {}}

        def frame(k, copy):
            bw, st = where[copy]
            outs = st.push([(StreamRecord(s.j, s.events[s.pos[copy]:]).set_state(*states[copy][s.j])
                             if states[copy].get(s.j) else StreamRecord(s.j, s.events[s.pos[copy]:])) for s in seqs])
            for s, o in zip(seqs, outs):
                s.pos[copy] += o["n_consumed"]
                assert len(o["frames"]) == 1 and o["frames"][0][0] == s.truth_t[k]
            if k == 0:
                return outs, None
            noise = seqs[0].run.truth.imu_noise
            tc = bw.track_camera([Camera(s.a, s.ta, k + 1, s.frames[k], s.K, min(k, 20), o["frames"][0][1],
                                         s.truth_t[k], noise, True) for s, o in zip(seqs, outs)], CAP,
                                 keypoint_distance=KD)
            for s, t in zip(seqs, tc):
                states[copy][s.j] = (s.truth_t[k], t["predicted"])
            slots = [s.a for s in seqs]
            if k % 4 == 3 or k == MOVE:
                bw.solve(slots, max_iterations=3)
            full = [s.a for s, t in zip(seqs, tc) if t["keyframe"] and bw.download([s.a], 4096)[0]["frames"].shape[0] >= 6]
            if full:
                bw.drop_victim(full)
            return outs, tc

        for k in range(MOVE + 1):
            frame(k, 1)
        # the checkpoint: the frame's state seated by a zero-event SET, then the three blobs
        st1.push([StreamRecord(s.j).set_state(*states[1][s.j]) for s in seqs])
        states[1] = {}
        jslots = [s.j for s in seqs]
        wblobs = bw1.save([s.a for s in seqs], [s.ta for s in seqs])
        sblobs = st1.save(jslots)
        assert all(_get(b, "drop_pending") == 1 and _get(b, "n2") > 0 for b in sblobs)
        bw2.restore([s.a for s in seqs], wblobs, [s.ta for s in seqs])
        st2.restore(jslots, sblobs)
        assert st2.save(jslots) == sblobs
        for s in seqs:
            s.pos[2] = s.pos[1]
        # the old way on the second handle's other slots: window and tracker blobs, the stream slot reset and fed
        # from the next reading
        bw2.restore([s.b for s in seqs], wblobs, [s.tb for s in seqs])
        old = [100 + s.j for s in seqs]
        st2.reset(old)
        old_outs = st2.push([StreamRecord(100 + s.j, s.events[s.pos[1]:]) for s in seqs])
        exact = inexact = 0
        fed_same = {s.j: True for s in seqs}
        for k in range(MOVE + 1, FRAMES + 1):
            o1, t1 = frame(k, 1)
            o2, t2 = frame(k, 2)
            for s, a, b in zip(seqs, o1, o2):
                assert a["n_consumed"] == b["n_consumed"]
                assert np.array_equal(_bits(a["frames"][0][1]), _bits(b["frames"][0][1]))
                if fed_same[s.j]:
                    assert np.array_equal(_bits(a["poses"]), _bits(b["poses"]))
            if k == MOVE + 1:                            # the old way's first released list is not the stream's
                for a, c in zip(o1, old_outs):
                    assert c["frames"] and c["frames"][0][0] == a["frames"][0][0]
                    ra, rc = a["frames"][0][1], c["frames"][0][1]
                    assert ra.shape != rc.shape or not np.array_equal(_bits(ra), _bits(rc))
            for s, x, y in zip(seqs, t1, t2):
                same = np.array_equal(_bits(x["predicted"]), _bits(y["predicted"]))
                fed_same[s.j] = fed_same[s.j] and same
                _same_frame(x, y, exact=False)
                exact += same
                inexact += not same
        print(f"moved at frame {MOVE}: {exact} frames bit-equal, {inexact} within the bar")
    finally:
        h1.close()
        h2.close()


def test_another_gpu(ba):
    torch = pytest.importorskip("torch")
    if torch.cuda.device_count() < 2:
        pytest.skip("one CUDA device")
    st = ImuStream(ba)
    seqs = [_Seq(s) for s in range(12)]
    slots = list(range(6000, 6012))
    st.reset(slots)
    for _ in range(10):
        live = [i for i, s in enumerate(seqs) if not s.done]
        for i, o in zip(live, st.push([seqs[i].record(slots[i]) for i in live])):
            seqs[i].took(o)
    blobs = st.save(slots)
    marks = [len(s.calls) for s in seqs]
    first = _drive(st, seqs, slots)
    with torch.cuda.device(1):
        c = BundleAdjustor(device=1, max_windows=1, max_frames=8, max_landmarks=64, max_obs=256)
        try:
            sc = ImuStream(c)
            sc.restore(slots, blobs)
            assert sc.save(slots) == blobs
            for s, slot, m, ref in zip(seqs, slots, marks, first):
                outs = []
                for ev, op in s.calls[m:]:                # the first pass's records on the other device
                    r = StreamRecord(slot, ev)
                    if op and op[0] == "set":
                        r.set_state(*op[1])
                    elif op:
                        r.clear_state()
                    outs.append(sc.push([r])[0])
                assert len(outs) == len(ref)
                for a, b in zip(outs, ref):
                    _equal_outs(a, b)
            assert sc.save(slots) == st.save(slots)
        finally:
            c.close()
