"""IMU stream slots of many sequences (include/pvio_b200.h "IMU stream slots", csrc/imu_stream.cu): per sequence the
IMU side of PVIO::Core on the device -- raw gyroscope and accelerometer readings synchronised into samples, samples
sorted into camera frames (with the prepend rule of the frontend applied), and the IMU-rate pose from the latest state
the caller feeds back."""
import numpy as np

from . import _lib

GYROSCOPE, ACCELEROMETER, CAMERA = _lib.IMU_EVENT_GYROSCOPE, _lib.IMU_EVENT_ACCELEROMETER, _lib.IMU_EVENT_CAMERA
KEEP, SET, CLEAR = _lib.IMU_STREAM_KEEP, _lib.IMU_STREAM_SET, _lib.IMU_STREAM_CLEAR
NO_STATE, NO_COVARIANCE = _lib.IMU_STREAM_NO_STATE, _lib.IMU_STREAM_NO_COVARIANCE


class StreamRecord:
    """One sequence's part of a push (pvio_b200_imu_stream_record): its stream slot, its new events as rows
    (kind, t, x, y, z) in arrival order, and optionally a new latest state (set_state: the 16-double `predicted` of
    track_camera with its frame time) or its removal (clear_state), applied before the events."""

    def __init__(self, slot, events=()):
        self.slot = int(slot)
        self.events = np.ascontiguousarray(np.asarray(events, dtype=np.float64).reshape(-1, 5))
        self.state_op, self.state_time, self.state = KEEP, 0.0, None

    def set_state(self, t, state16):
        self.state_op, self.state_time = SET, float(t)
        self.state = np.ascontiguousarray(state16, dtype=np.float64).reshape(16)
        return self

    def clear_state(self):
        self.state_op, self.state = CLEAR, None
        return self


class ImuStream:
    def __init__(self, ba):
        """ba: a BundleAdjustor (owns the device handle); stream slots are independent of its window slots."""
        self.ba, self.lib, self.h = ba, ba.lib, ba.h

    def reset(self, slots, output_q=None, output_p=None):
        """Empty each slot and clear its latest state; output_q [n, 4] xyzw / output_p [n, 3]: the output extrinsic
        (Config output_to_body_rotation / translation), identity when None."""
        s = np.ascontiguousarray(slots, dtype=np.int32).reshape(-1)
        n = len(s)
        q = np.tile([0.0, 0.0, 0.0, 1.0], (n, 1)) if output_q is None else output_q
        p = np.zeros((n, 3)) if output_p is None else output_p
        q = np.ascontiguousarray(np.broadcast_to(np.asarray(q, dtype=np.float64), (n, 4)))
        p = np.ascontiguousarray(np.broadcast_to(np.asarray(p, dtype=np.float64), (n, 3)))
        self.ba._ck(self.lib.pvio_b200_batch_imu_stream_reset(self.h, n, _lib.ptr(s), _lib.ptr(q), _lib.ptr(p)))

    def push(self, records):
        """One call over a list of StreamRecord (distinct slots).  Per record a dict: n_consumed (the events used, up to
        and including the first that released a frame), poses [n_consumed, 7] (q xyzw, p), frames: a list of
        (t, samples [k, 7]) for the released camera frames, samples as pvio_b200_window_camera takes them."""
        n = len(records)
        recs = (_lib.CImuStreamRecord * max(n, 1))()
        poses = []
        for r, rec in zip(recs, records):
            p = np.zeros((max(len(rec.events), 1), 7))
            poses.append(p)
            r.slot, r.n_events, r.state_op, r.state_time = rec.slot, len(rec.events), rec.state_op, rec.state_time
            _lib.set_ptrs(r, events=rec.events, state=rec.state, poses=p, rows=None)
        self.ba._ck(self.lib.pvio_b200_batch_imu_stream(self.h, n, recs))          # rows NULL: the sizes
        ft, fr, rows = [], [], []
        for r in recs[:n]:
            ft.append(np.zeros(max(r.need_frames, 1)))
            fr.append(np.zeros(max(r.need_frames, 1), dtype=np.int32))
            rows.append(np.zeros((max(r.need_rows, 1), 7)))
            r.max_frames, r.max_rows = r.need_frames, r.need_rows
            _lib.set_ptrs(r, frame_t=ft[-1], frame_rows=fr[-1], rows=rows[-1])
        self.ba._ck(self.lib.pvio_b200_batch_imu_stream(self.h, n, recs))
        out = []
        for i, r in enumerate(recs[:n]):
            frames, o = [], 0
            for k in range(r.n_frames):
                frames.append((float(ft[i][k]), rows[i][o:o + fr[i][k]].copy()))
                o += int(fr[i][k])
            out.append(dict(n_consumed=int(r.n_consumed), poses=poses[i][:r.n_consumed].copy(), frames=frames))
        return out

    def save(self, slots):
        """Save each stream slot to host memory.  Returns one blob (bytes) per slot, which restore() seats in any stream
        slot of any handle."""
        recs, n = self._snapshots(slots)
        self.ba._ck(self.lib.pvio_b200_batch_imu_stream_save(self.h, n, recs))     # data NULL: the sizes
        bufs = [np.zeros(recs[i].size, dtype=np.uint8) for i in range(n)]
        for i, b in enumerate(bufs):
            recs[i].data, recs[i].capacity = _lib.ptr(b), len(b)
        self.ba._ck(self.lib.pvio_b200_batch_imu_stream_save(self.h, n, recs))
        return [b.tobytes() for b in bufs]

    def restore(self, slots, blobs):
        """Restore blobs of save(): slot i takes blobs[i] and counts as reset.  One blob in several slots forks it."""
        recs, n = self._snapshots(slots)
        arrs = [np.frombuffer(b, dtype=np.uint8) for b in blobs]
        if len(arrs) != n:
            raise ValueError("one blob per slot")
        for i, a in enumerate(arrs):
            recs[i].data, recs[i].capacity = _lib.ptr(a), len(a)
        self.ba._ck(self.lib.pvio_b200_batch_imu_stream_restore(self.h, n, recs))

    def set_covariance(self, slots, state_times, covs, noise_cov, imu_records=None):
        """Give each slot's current latest state (its time state_times[i]) a covariance [15, 15] in [dtheta dp dv dbg dba],
        q perturbed on the right.  noise_cov [4, 9] (cov_w, cov_a, cov_bg, cov_ba), or one per slot: what predict()
        propagates with.  imu_records None (or a None entry): covs[i] is the state's own.  Otherwise imu_records[i] is the
        [288] factor returned with the `predicted` state and covs[i] the covariance of the frame it was predicted from.
        The seed holds until the slot's latest state changes."""
        slots = [int(s) for s in slots]
        n = len(slots)
        recs = (_lib.CImuStreamCovSeed * max(n, 1))()
        keep = []
        noise = np.broadcast_to(np.asarray(noise_cov, dtype=np.float64).reshape(-1, 36), (n, 36))
        for i, r in enumerate(recs[:n]):
            rec = None if imu_records is None else imu_records[i]
            c = np.ascontiguousarray(covs[i], dtype=np.float64).reshape(225)
            nz = np.ascontiguousarray(noise[i])
            ir = None if rec is None else np.ascontiguousarray(rec, dtype=np.float64).reshape(_lib.IMU_STRIDE)
            keep += [c, nz, ir]
            r.slot, r.state_time = slots[i], float(state_times[i])
            r.mode = _lib.IMU_STREAM_COV_DIRECT if ir is None else _lib.IMU_STREAM_COV_FACTOR
            _lib.set_ptrs(r, cov=c, noise_cov=nz, imu_record=ir)
        self.ba._ck(self.lib.pvio_b200_batch_imu_stream_set_covariance(self.h, n, recs))

    def predict(self, slots, times, states=False, covariances=True):
        """The IMU-rate pose of each slot at its non-decreasing times (times[i], one list per slot); changes no slot.
        Per slot a dict: status (0, NO_STATE or NO_COVARIANCE), poses [k, 7] (q xyzw, p) as the stream gives them,
        with states: states [k, 16]; with covariances: pose_cov [k, 6, 6] ([dtheta dp] of the pose) and state_cov
        [k, 15, 15], NaN without a seed."""
        slots = [int(s) for s in slots]
        n = len(slots)
        recs = (_lib.CImuStreamPredict * max(n, 1))()
        outs = []
        for i, r in enumerate(recs[:n]):
            t = np.ascontiguousarray(times[i], dtype=np.float64).reshape(-1)
            k = len(t)
            o = dict(times=t, poses=np.zeros((max(k, 1), 7)), states=np.zeros((max(k, 1), 16)) if states else None,
                     pose_cov=np.zeros((max(k, 1), 6, 6)) if covariances else None,
                     state_cov=np.zeros((max(k, 1), 15, 15)) if covariances else None)
            outs.append(o)
            r.slot, r.n_times = slots[i], k
            _lib.set_ptrs(r, times=t if k else None, poses=o["poses"], states=o["states"], pose_cov=o["pose_cov"],
                          state_cov=o["state_cov"])
        self.ba._ck(self.lib.pvio_b200_batch_imu_stream_predict(self.h, n, recs))
        res = []
        for r, o in zip(recs[:n], outs):
            k = len(o["times"])
            d = dict(status=int(r.status), poses=o["poses"][:k])
            if states:
                d["states"] = o["states"][:k]
            if covariances:
                d["pose_cov"], d["state_cov"] = o["pose_cov"][:k], o["state_cov"][:k]
            res.append(d)
        return res

    @staticmethod
    def _snapshots(slots):
        """the pvio_b200_imu_stream_snapshot records of a save / restore call, and their count"""
        slots = [int(s) for s in slots]
        recs = (_lib.CImuStreamSnapshot * max(len(slots), 1))()
        for r, s in zip(recs, slots):
            r.slot = s
        return recs, len(slots)
