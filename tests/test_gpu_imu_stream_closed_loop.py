"""pvio_b200_batch_imu_stream in front of pvio_b200_batch_window_track_camera, in lockstep: 8 inertial sequences over 21
camera frames.  Each sequence's raw IMU readings (gyroscope and accelerometer at 200 Hz with equal stamps) and camera
stamps go into its stream slot; each frame the stream releases goes through track_camera on window slot A with the
released sample list, and track_camera's `predicted` goes back into the stream slot as the latest state.  Keyframe
solves (from frame 3) and drops run on A.  The same loop runs on twin slot B with the sample lists, states and poses of
oracle/imu_stream_oracle.py built on the host (B takes A's window through save / restore after a solve or a drop, as
test_gpu_batch_window_track_camera does).  Checked every frame: the released lists and the IMU-rate poses bit for bit
against the oracle, every track_camera output and the save blobs of (A, TA) and (B, TB) bit for bit, and the IMU-rate
pose's motion over each frame against the synthetic ground truth's."""
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from oracle import imu_stream_oracle as so
from pvio_b200.batch_window import BatchWindows, Camera
from pvio_b200.bundle_adjustor import BundleAdjustor
from pvio_b200.imu_stream import ImuStream, StreamRecord
from test_gpu_batch_window_track_camera import CAP, KD, Seq, _bits, _same_blobs, _start, _take_a

pytestmark = pytest.mark.gpu
FRAMES = 21
# the IMU-rate pose at the frame's last sample, propagated from the previous frame's `predicted`: its motion since that
# state against the true motion between the two frames (DESIGN 4.7h)
ROT_TOL, POS_TOL = 0.01, 0.02              # rad, m
GRAVITY = np.array([0.0, 0.0, -so.GRAVITY])


def _motion(state, pose, dt, truth, k):
    """errors of the pose's motion since the state against the truth's from frame k - 1 to k, both in the body frame at
    the start: the rotation increment (rad) and the position increment less what the start velocity and gravity give
    (m).  The window's solves fit the test's rendered frames (a rotating camera over a textured plane, every track at
    unit inverse depth) rather than the synthetic trajectory, so the ground truth can check the motion over one frame,
    not the pose itself; and once a solve has moved the biases, the accelerometer bias it fitted moves the position
    increment away from the truth's (by about half the bias error times 0.25 s squared), so the position increment is
    held to the truth only on frames whose state still has the run's biases."""
    qs, qt0, qt1 = Rotation.from_quat(state[:4]), Rotation.from_quat(truth.q[k - 1]), Rotation.from_quat(truth.q[k])
    dr = ((qs.inv() * Rotation.from_quat(pose[:4])).inv() * (qt0.inv() * qt1)).magnitude()
    dp_pose = qs.inv().apply(pose[4:] - state[4:7] - state[7:10] * dt - 0.5 * GRAVITY * dt * dt)
    dp_true = qt0.inv().apply(truth.p[k] - truth.p[k - 1] - truth.v[k - 1] * dt - 0.5 * GRAVITY * dt * dt)
    return dr, np.linalg.norm(dp_pose - dp_true)


def _events(run):
    """arrival-ordered events: per sample a gyroscope then an accelerometer reading at its stamp, each camera stamp
    ahead of the readings at that time"""
    ev = []
    for k, (s, t_end) in enumerate(f[:2] for f in run.truth.imu_factors):
        for row in np.asarray(s):
            if k > 0 and row[0] == run.truth.imu_factors[k - 1][1]:
                ev.append((so.CAMERA, row[0], 0.0, 0.0, 0.0))
            elif k == 0 and row[0] == 0.0:
                ev.append((so.CAMERA, 0.0, 0.0, 0.0, 0.0))
            ev.append((so.GYROSCOPE, row[0], *row[1:4]))
            ev.append((so.ACCELEROMETER, row[0], *row[4:7]))
    return np.array(ev, dtype=np.float64)


def _sincos_device():
    """the device's sin / cos (torch on the same GPU), computed on demand, so the oracle's poses are the device's bits"""
    import torch
    table = {}

    def sincos(v):
        if v not in table:
            y = torch.tensor([v], dtype=torch.float64, device="cuda")
            table[v] = (torch.sin(y).item(), torch.cos(y).item())
        return table[v]
    return sincos


@pytest.fixture(scope="module")
def ba():
    b = BundleAdjustor(max_windows=16, max_frames=9, max_landmarks=4096, max_obs=16384)
    yield b
    b.close()


def test_stream_track_camera_loop_equals_the_host_built_loop(ba):
    bw, st = BatchWindows(ba), ImuStream(ba)
    seqs = [Seq(j, j, 8 + j, FRAMES + 3, 1700 + j) for j in range(8)]
    _start(bw, seqs)
    sincos = _sincos_device()
    for s in seqs:
        s.events, s.pos, s.state = _events(s.run), 0, None
        s.oracle = so.Stream(sincos=sincos)
        s.truth_t = [0.0] + [f[1] for f in s.run.truth.imu_factors]
    st.reset([s.j for s in seqs])
    checked_poses = checked_pos = solved = dropped = 0
    rot_err = pos_err = 0.0
    for k in range(FRAMES + 1):
        # stream until every sequence releases its next frame (the sequences share one timing, so they do together)
        outs = st.push([(StreamRecord(s.j, s.events[s.pos:]).set_state(*s.state) if s.state
                         else StreamRecord(s.j, s.events[s.pos:])) for s in seqs])
        for s, o in zip(seqs, outs):
            poses, n, rel = s.oracle.push(s.events[s.pos:], state=s.state)
            assert o["n_consumed"] == n
            assert np.array_equal(_bits(o["poses"]), _bits(np.array(poses).reshape(-1, 7)))
            assert len(o["frames"]) == len(rel) == 1
            (t, rows), (rt, rrows) = o["frames"][0], rel[0]
            assert t == rt == s.truth_t[k]
            s.rows_b = np.array(rrows, dtype=np.float64)
            assert np.array_equal(_bits(rows), _bits(s.rows_b))
            s.rows_a = rows
            if s.state is not None:              # the motion since the state against the truth's (_motion)
                (i,) = np.flatnonzero((s.events[s.pos:s.pos + n, 0] == so.ACCELEROMETER)
                                      & (s.events[s.pos:s.pos + n, 1] == s.truth_t[k]))
                dr, dp = _motion(s.state[1], o["poses"][i], s.truth_t[k] - s.state[0], s.run.truth, k)
                rot_err = max(rot_err, dr)
                checked_poses += 1
                if s.state_unsolved:                 # the state's biases are still the synthetic run's guess
                    pos_err = max(pos_err, dp)
                    checked_pos += 1
            s.pos += n
        if k == 0:                               # the sequence start: the window and tracker slots already hold it
            continue
        for s in seqs:
            s.f += 1
            assert s.f == k
        noise = seqs[0].run.truth.imu_noise
        cam = lambda s, slot, tr, rows: Camera(slot, tr, s.f + 1, s.frames[s.f], s.K, min(s.f, 20), rows,   # noqa: E731
                                              s.truth_t[k], noise, True)
        oa = bw.track_camera([cam(s, s.a, s.ta, s.rows_a) for s in seqs], CAP, keypoint_distance=KD)
        ob = bw.track_camera([cam(s, s.b, s.tb, s.rows_b) for s in seqs], CAP, keypoint_distance=KD)
        for a, b in zip(oa, ob):
            assert a["n_keypoints"] == b["n_keypoints"]
            for key in ("keypoints", "state", "predicted", "imu_record", "predict_q", "parallax"):
                assert np.array_equal(_bits(a[key]), _bits(b[key])), key
            for key in ("prev_index", "kp_track", "counts", "feature_counts", "info"):
                assert np.array_equal(a[key], b[key]), key
            for key in ("keyframe", "n_parallax", "skipped_frames"):
                assert a[key] == b[key], key
        _same_blobs(bw, seqs, k)
        for s, a, b in zip(seqs, oa, ob):
            s.newest_kf = a["keyframe"]
            s.state = (s.truth_t[k], a["predicted"])
            s.state_unsolved = solved == 0
            assert np.array_equal(_bits(a["predicted"]), _bits(b["predicted"]))
        took = False
        if k % 4 == 3:
            bw.solve([s.a for s in seqs], max_iterations=3)
            solved += 1
            took = True
        full = [s for s in seqs if s.newest_kf and bw.download([s.a], 4096)[0]["frames"].shape[0] >= 6]
        if full:
            bw.drop_victim([s.a for s in full])
            dropped += len(full)
            took = True
        if took:
            _take_a(bw, seqs)
        _same_blobs(bw, seqs, k)
    print(f"closed loop: {FRAMES} frames x {len(seqs)} sequences, solves {solved}, drops {dropped}, pose motion against the "
          f"truth: rotation error <= {rot_err:.2e} rad over {checked_poses} frames, position <= {pos_err:.2e} m over "
          f"{checked_pos} frames before the first solve")
    assert solved > 0 and dropped > 0 and checked_poses == len(seqs) * (FRAMES - 1) and checked_pos == 3 * len(seqs)
    assert rot_err < ROT_TOL and pos_err < POS_TOL
