"""pvio_b200_batch_window_localize: the per-camera-frame half of SlidingWindowTracker::track on resident slots -- the PnP
of the new frame against the slot's own landmarks, and the triangulation of the tracks born in it -- without the host
mirroring any landmark.  Checked against a host gather from the slot download, against pvio_b200_batch_pnp_solve and
pvio_b200_triangulate fed from that gather, against the fp64 oracles, and along whole sequences."""
import ctypes as C

import numpy as np
import pytest

from oracle import pnp_oracle as po
from oracle import tri_oracle as to
from pvio_b200 import _lib, triangulate
from pvio_b200.pnp import imu_record
from pvio_b200.batch_window import Edit, Localize
from pvio_b200.bundle_adjustor import BundleAdjustor, PvioB200Error
from pvio_b200._lib import EINVAL
from synthetic import so3
from synthetic.sequence import BatchPlayer, Run

pytestmark = pytest.mark.gpu
COST_TOL, STATE_TOL = 1e-9, 1e-8          # the bars of test_gpu_pnp.py
SEQ_TOL = 2e-6                            # the bar of the resident sequence tests


# ------------------------------------------------------------------------ helpers
def _state16(run, f):
    g = run.guess
    return np.concatenate([g.q[f], g.p[f], g.v[f], g.bg[f], g.ba[f]])


def _given_point(run, l):
    """a fixed world point for a track of a plane role (the shim's plane-cast point): its first ray at rho0"""
    fr, zs = run.tracks[l]
    qc, pc = run.cam_pose(run.guess.q[fr[0]], run.guess.p[fr[0]])
    return so3.qrot(qc, np.array([zs[0][0], zs[0][1], 1.0]) / run.rho0[l]) + pc


def _record(player, j, f, newest_abs, perturb=1e-3, inertial=True, born=True):
    """the Localize of absolute frame f of run j: its keypoints on the live tracks (a point for plane roles) and the
    tracks observed in newest_abs and f that are not live.  Returns (record, observed landmarks, new landmarks)."""
    run = player.runs[j]
    s = _state16(run, f).copy()
    s[4:7] += perturb
    L = Localize(player.slots[j], s, player.rec[j][f - 1] if inertial else None)
    obs_l, new_l = [], []
    for l, (fr, zs) in enumerate(run.tracks):
        if f not in fr:
            continue
        z = zs[fr.index(f)]
        if l in player.ids[j]:
            L.observe(player.ids[j][l], z, _given_point(run, l) if player.roles[j].get(l, -1) != -1 else None)
            obs_l.append(l)
        elif born and newest_abs in fr:
            L.born(zs[fr.index(newest_abs)], z)
            new_l.append(l)
    return L, obs_l, new_l


def _host_points(run, d, win, L, obs_l, newest_abs):
    """Track::get_landmark_point from a slot download (win: the absolute frame of each window frame), or the given
    point; NaN for a track not observed in the newest frame"""
    row = {int(t): r for r, t in enumerate(d["ids"])}
    out = np.full((len(obs_l), 3), np.nan)
    for i, (l, (tid, _, pt)) in enumerate(zip(obs_l, L.obs)):
        fr, zs = run.tracks[l]
        if newest_abs not in fr:
            continue
        if pt is not None:
            out[i] = pt
            continue
        r = row[tid]
        a = int(d["anchor"][r])
        qc, pc = run.cam_pose(d["frames"][a, 0:4], d["frames"][a, 4:7])
        za = zs[fr.index(win[a])]
        out[i] = so3.qrot(qc, np.array([za[0], za[1], 1.0]) / d["inv_depth"][r]) + pc
    return out


def _host_pnp(ba, problems, max_iterations=10):
    """pvio_b200_batch_pnp_solve of (run, last16, record, points) problems: the rows with a point take part"""
    n = len(problems)
    pbs, keep = (_lib.CPnpProblem * n)(), []
    frames = np.zeros((n, 16))
    for i, (run, last, L, pts) in enumerate(problems):
        w, pb = run.w, pbs[i]
        ok = ~np.isnan(pts[:, 0]) if len(pts) else np.zeros(0, dtype=bool)
        x = np.ascontiguousarray(pts[ok], dtype=np.float64).reshape(-1, 3)
        z = np.ascontiguousarray([o[1] for o, k in zip(L.obs, ok) if k], dtype=np.float64).reshape(-1, 2)
        lf = np.ascontiguousarray(last, dtype=np.float64)
        rec = L.imu if L.imu is not None else np.zeros(_lib.IMU_STRIDE)
        keep += [x, z, lf, rec]
        pb.n_points, pb.use_inertial = len(x), 0 if L.imu is None else 1
        pb.points, pb.z = _lib.ptr(x), _lib.ptr(z)
        pb.cam_q_cs[:], pb.cam_p_cs[:] = list(w.cam_q_cs), list(w.cam_p_cs)
        pb.imu_q_cs[:], pb.imu_p_cs[:] = list(w.imu_q_cs), list(w.imu_p_cs)
        pb.sqrt_inv_cov[:] = list(np.asarray(w.sqrt_inv_cov, dtype=np.float64).reshape(4))
        pb.cauchy_a = w.cauchy_a
        pb.last_frame, pb.imu_data = _lib.ptr(lf), _lib.ptr(rec)
        frames[i] = L.state
    opt = _lib.COptions(max_iterations, 1e6, 1, 0, 0.0)
    sms = (_lib.CSummary * n)()
    ba._ck(ba.lib.pvio_b200_batch_pnp_solve(ba.h, n, pbs, _lib.ptr(frames), 16, C.byref(opt), sms))
    return frames, [_lib.summary(sms[i]) for i in range(n)]


def _cam_matrix(run, x16):
    qc, pc = run.cam_pose(x16[0:4], x16[4:7])
    return to.projection_matrix(qc, pc), qc, pc


def _host_triangulate(ba, run, last16, new16, L):
    """pvio_b200_triangulate over the two host-built camera matrices; (valid, points, rho, rho_next, oracle results)"""
    T = len(L.new)
    Pa, qa, pa = _cam_matrix(run, last16)
    Pn, qn, pn = _cam_matrix(run, new16)
    z = np.array([[a, b] for a, b in L.new], dtype=np.float64).reshape(-1, 2)
    pts, valid, _ = triangulate.triangulate(ba, np.stack([Pa, Pn]), np.arange(0, 2 * T + 1, 2), np.tile([0, 1], T), z)
    rho, nxt = np.full(T, np.nan), np.full(T, np.nan)
    for t in range(T):
        if valid[t]:
            rho[t] = 1.0 / so3.qrot(so3.qconj(qa), pts[t] - pa)[2]
            nxt[t] = _reanchor(qa, pa, qn, pn, L.new[t][0], rho[t])
    oracle = [to.triangulate_scored([Pa, Pn], [a, b]) for a, b in L.new]
    return valid, pts, rho, nxt, oracle, (Pa, Pn)


def _reanchor(qa, pa, qn, pn, z, rho):
    """Chain._reanchor's formula: the inverse depth in camera (qa, pa) re-expressed in camera (qn, pn)"""
    x = so3.qrot(qa, np.array([z[0], z[1], 1.0]) / rho) + pa
    return 1.0 / so3.qrot(so3.qconj(qn), x - pn)[2]


def _near_threshold(P2, z2, eps=1e-9):
    """a case whose parallax / depth test is within eps of its threshold (excluded from the validity comparison)"""
    A = np.vstack([[z[0] * P[2] - P[0], z[1] * P[2] - P[1]] for P, z in zip(P2, z2)])
    q = np.linalg.svd(A)[2][3]
    for P in P2:
        qi = P @ q
        if abs(qi[2] * q[3]) <= eps * abs(qi[2]) * abs(q[3]) + 1e-300 or abs(qi[2] / q[3] - 100.0) <= eps * 100.0:
            return True
    return False


def _downloads(bw, slots, stride):
    return [{k: v.copy() for k, v in d.items()} for d in bw.download(slots, stride)]


def _same_download(a, b):
    return all(np.array_equal(x[k], y[k], equal_nan=True) for x, y in zip(a, b) for k in x)


RUNS = [dict(F=20, N=6, M=220, seed=720), dict(F=20, N=8, M=240, seed=722, planes=2), dict(F=20, N=9, M=260, seed=724)]


@pytest.fixture(scope="module")
def setup():
    """four resident slots (the second with plane tracks) after their first solve; slot 4 is not resident and slot 5 is
    resident without frames"""
    runs = [Run(**kw) for kw in RUNS]
    ba = BundleAdjustor(max_windows=6, max_frames=9, max_landmarks=400, max_obs=3000)
    player = BatchPlayer(ba, runs + [Run(F=20, N=6, M=220, seed=726)])
    player.bw.reset(5, runs[0].w)
    # the tracks first seen in the newest frame leave again: they are born in the next frame (keypoints in both), and
    # their ids are dead
    edits, player.dead = [], []
    for j, r in enumerate(player.runs):
        e = Edit(player.slots[j])
        e.remove = [player.ids[j].pop(l) for l in sorted(player.ids[j]) if r.tracks[l][0][0] == r.N - 1]
        player.dead.append(list(e.remove))
        edits.append(e)
    player.bw.edit(edits)
    player.model.edit(edits)
    player.bw.solve(list(range(4)), max_iterations=4)
    yield ba, player
    ba.close()


def _frame_records(player, js, perturb=1e-3):
    out = []
    for j in js:
        run = player.runs[j]
        f = player.k[j] + run.N
        out.append(_record(player, j, f, f - 1, perturb=perturb))
    return out


# ------------------------------------------------------------------------ 1, 5: gather, plane points, slots untouched
def test_gather_matches_the_host_gather_and_leaves_every_slot_untouched(setup):
    ba, player = setup
    js = [0, 1, 2]
    recs = _frame_records(player, js)
    # a live track that is not observed in the newest frame takes no part: its row is NaN
    for (L, obs_l, _), j in zip(recs, js):
        run, f_new = player.runs[j], player.k[j] + player.runs[j].N - 1
        extra = next(l for l in sorted(player.ids[j]) if f_new not in run.tracks[l][0] and l not in obs_l)
        L.observe(player.ids[j][extra], [0.01, -0.02])
        obs_l.append(extra)
    assert any(p is not None for p in (o[2] for o in recs[1][0].obs))          # the plane run names plane points
    before = _downloads(player.bw, [0, 1, 2, 3, 5], 400)
    out = player.bw.localize([r[0] for r in recs])
    after = _downloads(player.bw, [0, 1, 2, 3, 5], 400)
    assert _same_download(before, after)
    used_given = 0
    for (L, obs_l, _), j, o, d in zip(recs, js, out, before):
        run = player.runs[j]
        ref = _host_points(run, d, list(range(player.k[j], player.k[j] + run.N)), L, obs_l, player.k[j] + run.N - 1)
        assert np.array_equal(np.isnan(ref[:, 0]), np.isnan(o["points"][:, 0]))
        assert np.isnan(o["points"][-1]).all()
        ok = ~np.isnan(ref[:, 0])
        assert ok.sum() > 20
        err = np.abs(o["points"][ok] - ref[ok]).max(axis=1) / np.abs(ref[ok]).max(axis=1)
        assert err.max() <= 1e-12, err.max()
        for i, (_, _, pt) in enumerate(L.obs):
            if pt is not None and ok[i]:
                assert np.array_equal(o["points"][i], pt)
                used_given += 1
    assert used_given > 0                                      # plane-role rows took part with their given points


# ------------------------------------------------------------------------ 2, 3: PnP as batch_pnp_solve, oracle
@pytest.mark.parametrize("js", [[1], [0, 1, 2]], ids=["n1", "n3"])
def test_pnp_equals_batch_pnp_solve_and_the_oracle(setup, js):
    """pnp_kernel combines its warps with shared-memory atomics, so two runs of one problem may differ in the last bits
    (DESIGN 4.6), even after several runs agreed bit for bit: localize and batch_pnp_solve of the same problem agree to
    rounding -- the same iterations, accepted steps, termination and usability, costs and states within 1e-12."""
    ba, player = setup
    recs = _frame_records(player, js, perturb=2e-3)
    ds = player.bw.download([player.slots[j] for j in js], 400)
    out = player.bw.localize([r[0] for r in recs])
    probs = [(player.runs[j], d["frames"][-1], L, o["points"]) for j, d, (L, _, _), o in zip(js, ds, recs, out)]
    xs, sms = _host_pnp(ba, probs)
    for (run, last, L, pts), o, x, sm in zip(probs, out, xs, sms):
        for k in ("iterations", "accepted_steps", "termination", "usable"):
            assert o["summary"][k] == sm[k], k
        for k in ("initial_cost", "final_cost"):
            assert abs(o["summary"][k] - sm[k]) <= 1e-12 * abs(sm[k]), k
        assert np.abs(o["state"] - x).max() <= 1e-12 * max(np.abs(x).max(), 1.0)
        assert o["summary"]["iterations"] > 0 and o["summary"]["solve_seconds"] > 0
        ok = ~np.isnan(pts[:, 0])
        r = L.imu
        imu = dict(dt=r[0], dq=r[1:5], dp=r[5:8], dv=r[8:11], sqrt_inv_cov=r[11:236].reshape(15, 15),
                   dq_dbg=r[236:245].reshape(3, 3), dp_dbg=r[245:254].reshape(3, 3), dp_dba=r[254:263].reshape(3, 3),
                   dv_dbg=r[263:272].reshape(3, 3), dv_dba=r[272:281].reshape(3, 3))
        w = run.w
        xr, sr = po.pnp_solve(L.state, last, imu, pts[ok], np.array([ob[1] for ob in L.obs])[ok], w.cam_q_cs, w.cam_p_cs,
                              w.imu_q_cs, w.imu_p_cs, w.sqrt_inv_cov, True, cauchy_a=w.cauchy_a)
        assert o["summary"]["iterations"] == sr["iterations"]
        assert abs(o["summary"]["initial_cost"] - sr["initial_cost"]) <= COST_TOL * sr["initial_cost"]
        assert abs(o["summary"]["final_cost"] - sr["final_cost"]) <= COST_TOL * sr["final_cost"]
        assert np.linalg.norm(o["state"] - xr) < STATE_TOL * max(np.linalg.norm(xr - L.state), 1e-3)


# ------------------------------------------------------------------------ 4: triangulation
CASES = ((-4.0, 0.1), (-1.5, -0.2), (150.0, 0.05), (400.0, -0.1), (30.0, 0.02))    # (depth, ray offset): behind, far, near


def test_triangulation_matches_the_oracle_and_the_triangulate_call(setup):
    ba, player = setup
    recs = _frame_records(player, [0, 2])
    ds = player.bw.download([0, 2], 400)
    for (L, _, _), j, d in zip(recs, [0, 2], ds):
        run = player.runs[j]
        qa, pa = run.cam_pose(d["frames"][-1, 0:4], d["frames"][-1, 4:7])
        for depth, side in CASES:
            x = so3.qrot(qa, np.array([side, 0.5 * side, 1.0]) * depth) + pa       # behind the camera, far, near
            zl = so3.qrot(so3.qconj(qa), x - pa)
            qn, pn = run.cam_pose(L.state[0:4], L.state[4:7])
            zn = so3.qrot(so3.qconj(qn), x - pn)
            L.born(zl[:2] / zl[2], zn[:2] / zn[2])
    out = player.bw.localize([r[0] for r in recs])
    checked, kinds = 0, set()
    for (L, _, _), j, d, o in zip(recs, [0, 2], ds, out):
        run = player.runs[j]
        valid, pts, rho, nxt, oracle, Ps = _host_triangulate(ba, run, d["frames"][-1], o["state"], L)
        assert len(L.new) > 10
        for t in range(len(L.new)):
            if _near_threshold(Ps, L.new[t]):
                continue
            checked += 1
            assert o["valid"][t] == valid[t] == oracle[t][0], t
            if not valid[t]:
                kinds.add("behind" if t >= len(L.new) - 5 and CASES[t - len(L.new) + 5][0] < 0 else
                          "far" if t >= len(L.new) - 5 and CASES[t - len(L.new) + 5][0] >= 100 else "other")
                assert np.isnan(o["inv_depth"][t]) and np.isnan(o["inv_depth_next"][t])
                continue
            qa, pa = run.cam_pose(d["frames"][-1, 0:4], d["frames"][-1, 4:7])
            qn, pn = run.cam_pose(o["state"][0:4], o["state"][4:7])
            rho_oracle = 1.0 / so3.qrot(so3.qconj(qa), oracle[t][1] - pa)[2]
            assert np.linalg.norm(pts[t] - oracle[t][1]) <= 1e-9 * np.linalg.norm(oracle[t][1])
            assert abs(o["inv_depth"][t] - rho[t]) <= 1e-9 * abs(rho[t])
            assert abs(o["inv_depth"][t] - rho_oracle) <= 1e-9 * abs(rho_oracle)
            ref = _reanchor(qa, pa, qn, pn, L.new[t][0], o["inv_depth"][t])
            assert abs(o["inv_depth_next"][t] - ref) <= 1e-12 * abs(ref)
    print(f"{checked} tracks compared, invalid kinds: {sorted(kinds)}")
    assert checked > 20 and {"behind", "far"} <= kinds


# ------------------------------------------------------------------------ 6: rejections
def _spoil_slot(recs, keep, player):
    recs[1].slot = 77


def _spoil_twice(recs, keep, player):
    recs[1].slot = recs[0].slot


def _spoil_not_resident(recs, keep, player):
    recs[1].slot = 4


def _spoil_no_frames(recs, keep, player):
    recs[1].slot = 5


def _spoil_dead(recs, keep, player):
    assert player.dead[1]
    t = np.ctypeslib.as_array(recs[1].obs_track, shape=(recs[1].n_obs,)).copy()
    t[0] = player.dead[1][0]                              # a removed track of the slot
    keep.append(t)
    recs[1].obs_track = _lib.ptr(t)


def _spoil_unknown(recs, keep, player):
    t = np.array([10 ** 6], dtype=np.int32)
    keep.append(t)
    recs[1].obs_track = _lib.ptr(t)
    recs[1].n_obs = 1


def _spoil_track_twice(recs, keep, player):
    t = np.ctypeslib.as_array(recs[1].obs_track, shape=(recs[1].n_obs,)).copy()
    t[3] = t[2]
    keep.append(t)
    recs[1].obs_track = _lib.ptr(t)


def _spoil_z(recs, keep, player):
    z = np.ctypeslib.as_array(recs[1].obs_z, shape=(recs[1].n_obs, 2)).copy()
    z[4, 1] = np.inf
    keep.append(z)
    recs[1].obs_z = _lib.ptr(z)


def _spoil_new_z(recs, keep, player):
    z = np.ctypeslib.as_array(recs[0].new_z, shape=(recs[0].n_new, 2)).copy()
    z[0, 0] = np.nan
    keep.append(z)
    recs[0].new_z = _lib.ptr(z)


def _spoil_null(recs, keep, player):
    recs[0].new_inv_depth = None


def _spoil_state(recs, keep, player):
    recs[1].state = None


def _spoil_imu(recs, keep, player):
    recs[1].imu_record = None


def _spoil_plane_point(recs, keep, player):
    x = np.full((recs[1].n_obs, 3), np.nan)               # the plane run without its plane-cast points
    keep.append(x)
    recs[1].obs_point = _lib.ptr(x)


SPOILERS = [_spoil_slot, _spoil_not_resident, _spoil_no_frames, _spoil_twice, _spoil_dead, _spoil_unknown,
            _spoil_track_twice, _spoil_z, _spoil_new_z, _spoil_null, _spoil_state, _spoil_imu, _spoil_plane_point]


@pytest.mark.parametrize("spoil", SPOILERS, ids=[s.__name__[7:] for s in SPOILERS])
def test_rejections_change_no_output(setup, spoil):
    ba, player = setup
    built = _frame_records(player, [0, 1])
    keep, n = [], 2
    recs = (_lib.CWindowLocalize * n)()
    outs = []
    for r, (L, _, _) in zip(recs, built):
        t = np.array([o[0] for o in L.obs], dtype=np.int32)
        z = np.array([o[1] for o in L.obs], dtype=np.float64).reshape(-1, 2)
        x = np.array([np.full(3, np.nan) if o[2] is None else o[2] for o in L.obs]).reshape(-1, 3)
        zl = np.array([a for a, _ in L.new]).reshape(-1, 2)
        zn = np.array([b for _, b in L.new]).reshape(-1, 2)
        o = dict(state=np.full(16, 7.0), points=np.full((len(t), 3), 7.0), valid=np.full(len(zl), 7, dtype=np.uint8),
                 rho=np.full(len(zl), 7.0), nxt=np.full(len(zl), 7.0))
        keep += [t, z, x, zl, zn, L.imu]
        outs.append(o)
        sm = _lib.CSummary()
        sm.iterations = 777
        o["sm"] = sm
        r.slot, r.use_inertial, r.imu_record = L.slot, 1, _lib.ptr(L.imu)
        r.state = _lib.ptr(o["state"])
        r.n_obs, r.obs_track, r.obs_z, r.obs_point = len(t), _lib.ptr(t), _lib.ptr(z), _lib.ptr(x)
        r.points_out = _lib.ptr(o["points"])
        r.n_new, r.new_z_last, r.new_z = len(zl), _lib.ptr(zl), _lib.ptr(zn)
        r.new_valid, r.new_inv_depth = _lib.ptr(o["valid"]), _lib.ptr(o["rho"])
        r.new_inv_depth_next, r.summary = _lib.ptr(o["nxt"]), C.pointer(sm)
    assert recs[0].n_new > 0 and recs[1].n_obs > 5
    spoil(recs, keep, player)
    before = _downloads(player.bw, [0, 1, 2, 3, 5], 400)
    n0 = ba.kernel_launches
    rc = ba.lib.pvio_b200_batch_window_localize(ba.h, n, recs, None)
    assert rc == EINVAL
    assert ba.kernel_launches == n0
    for o in outs:
        assert np.all(o["state"] == 7.0) and np.all(o["points"] == 7.0) and np.all(o["valid"] == 7)
        assert np.all(o["rho"] == 7.0) and np.all(o["nxt"] == 7.0) and o["sm"].iterations == 777
    assert _same_download(before, _downloads(player.bw, [0, 1, 2, 3, 5], 400))
    player.bw.localize([b[0] for b in built])                  # the handle is still usable


# ------------------------------------------------------------------------ 7: launch count
def test_three_launches_whatever_n(setup):
    ba, player = setup
    for js in ([0], [0, 1, 2, 3]):
        recs = [r[0] for r in _frame_records(player, js)]
        n0 = ba.kernel_launches
        player.bw.localize(recs)
        assert ba.kernel_launches - n0 == 3
    n0 = ba.kernel_launches
    assert player.bw.localize([]) == [] and ba.kernel_launches == n0
    with pytest.raises(PvioB200Error):
        player.bw.localize([Localize(player.slots[0], np.zeros(16)), Localize(player.slots[0], np.zeros(16))])


# ------------------------------------------------------------------------ 8: sequences
def _z(run, l, f):
    fr, zs = run.tracks[l]
    return zs[fr.index(f)]


def _merged_record(run, g):
    """the IMU record from absolute frame g - 2 to g when frame g - 1 is erased: the samples of both factors integrated
    at the biases of g - 2 (sliding_window_tracker.cpp:115-119)"""
    (s0, _, bg, ba), (s1, t1, _, _) = run.truth.imu_factors[g - 2], run.truth.imu_factors[g - 1]
    pre = so3.PreIntegrator(*run.truth.imu_noise)
    pre.data = [(r[0], r[1:4], r[4:7]) for r in np.concatenate([s0, s1])]
    rec = imu_record(pre.integrate(t1, bg, ba))
    rec[281:284], rec[284:287] = bg, ba
    return rec


class _Path:
    """One way of running the per-camera-frame cycle on the slots of a BatchPlayer: `device` takes each frame's state
    and new inverse depths from localize, otherwise from a host gather of the download + batch_pnp_solve +
    pvio_b200_triangulate.  win[j]: the absolute frame of each window frame of slot j."""

    def __init__(self, ba, runs, slots, device):
        self.ba, self.device = ba, device
        self.p = BatchPlayer(ba, runs, slots=slots)
        self.win = [list(range(r.N)) for r in runs]

    def localize(self, built, newest_abs):
        p = self.p
        js = list(range(len(built)))
        if self.device:
            out = p.bw.localize([b[0] for b in built])
            return [(o["state"], o["summary"], o["valid"], o["inv_depth"], o["inv_depth_next"]) for o in out]
        ds = p.bw.download(p.slots, 400)
        probs = []
        for j, d, (L, obs_l, _) in zip(js, ds, built):
            pts = _host_points(p.runs[j], d, self.win[j], L, obs_l, newest_abs[j])
            probs.append((p.runs[j], d["frames"][-1], L, pts))
        xs, sms = _host_pnp(self.ba, probs)
        res = []
        for j, d, (L, _, _), x, sm in zip(js, ds, built, xs, sms):
            if L.new:
                valid, _, rho, nxt, _, _ = _host_triangulate(self.ba, p.runs[j], d["frames"][-1], x, L)
            else:
                valid, rho, nxt = np.zeros(0, dtype=bool), np.zeros(0), np.zeros(0)
            res.append((x, sm, valid, rho, nxt))
        return res

    def append(self, built, res, fs, replace=False):
        """the frame edit of absolute frames fs: the new frame at its solved state with the observations of the live
        tracks, and the valid new tracks -- after a keyframe at the slot's newest frame with inv_depth (their
        observations in the new frame follow in a second edit); replacing a non-keyframe (replace_last), at the new
        frame with inv_depth_next and the IMU record from the frame before the erased one"""
        p = self.p
        edits, born = [], []
        for j, ((L, obs_l, new_l), (x, _, valid, rho, nxt)) in enumerate(zip(built, res)):
            run, N, f = p.runs[j], p.runs[j].N, fs[j]
            e = Edit(p.slots[j], replace).frame(x, False, _merged_record(run, f) if replace else p.rec[j][f - 1])
            for l in obs_l:
                e.obs.append((p.ids[j][l], N - 1, _z(run, l, f)))
            for (zl, zn), v, r, rn in zip(L.new, valid, rho, nxt):
                if v:
                    e.new.append((N - 1, zn, rn) if replace else (N - 2, zl, r))
            edits.append(e)
            born.append([l for l, v in zip(new_l, valid) if v])
        got = p.bw.edit(edits)
        p.model.edit(edits)
        follow = []
        for j, (ls, ids) in enumerate(zip(born, got)):
            e = Edit(p.slots[j])
            for l, i in zip(ls, ids):
                p.ids[j][l], p.roles[j][l] = int(i), -1
                if not replace:
                    e.obs.append((int(i), p.runs[j].N - 1, _z(p.runs[j], l, fs[j])))
            follow.append(e)
            if replace:
                self.win[j][-1] = fs[j]
            else:
                self.win[j].append(fs[j])
        if not replace:
            p.bw.edit(follow)
            p.model.edit(follow)


def test_sequences_follow_the_host_path():
    """4 inertial sequences (N = 6, 8, 9, 6; the second with planes) take 11 keyframes; after every other keyframe the
    next frame is a non-keyframe that the frame after it replaces (replace_last, its new tracks anchored in the new
    frame with inv_depth_next, the IMU record merged over the erased frame).  Each frame's state comes from localize
    (from a perturbed prediction) and each new track's inverse depth from its triangulation; a host path over the same
    inputs (download, host gather, batch_pnp_solve, pvio_b200_triangulate) drives slots 4 .. 7 and must give the same
    iterations and landmarks and the same states within the bar of the resident sequence tests."""
    kws = [dict(F=23, N=6, M=220, seed=730), dict(F=25, N=8, M=260, seed=732, planes=2),
           dict(F=26, N=9, M=260, seed=734), dict(F=23, N=6, M=220, seed=736)]
    ba = BundleAdjustor(max_windows=8, max_frames=9, max_landmarks=400, max_obs=3000)
    paths = [_Path(ba, [Run(**kw) for kw in kws], list(range(4)), True),
             _Path(ba, [Run(**kw) for kw in kws], list(range(4, 8)), False)]
    worst, replaced, anchored_next = 0.0, 0, 0
    for step in range(11):
        nonkey = step % 2 == 1
        outs = []
        for P in paths:
            p = P.p
            sms = p.bw.solve(p.slots, max_iterations=10)            # the reference's solver_iteration_limit
            fs = [w[-1] + 1 for w in P.win]
            built = [_record(p, j, f, f - 1, perturb=3e-3 if nonkey else 1e-3) for j, f in enumerate(fs)]
            res = P.localize(built, [f - 1 for f in fs])
            p.bw.drop_victim(p.slots)
            p.model.drop_victim(p.slots)
            p.refresh(list(range(4)), 400)
            for j in range(4):
                p.k[j] += 1
                P.win[j].pop(0)
            P.append(built, res, fs)
            seq = [(sms, res)]
            if nonkey:                           # frame f + 1 replaces the non-keyframe f
                gs = [f + 1 for f in fs]
                built2 = [_record(p, j, g, g - 1) for j, g in enumerate(gs)]
                p.refresh(list(range(4)), 400)
                res2 = P.localize(built2, fs)
                P.append(built2, res2, gs, replace=True)
                seq.append((None, res2))
                anchored_next += sum(int(np.sum(r[2])) for r in res2) if P.device else 0
            p.refresh(list(range(4)), 400)
            p.set_roles(list(range(4)))
            outs.append((seq, {j: dict(p.ids[j]) for j in range(4)}))
        (sd, ids_d), (sh, ids_h) = outs
        assert ids_d == ids_h, step
        for (sm_d, rd), (sm_h, rh) in zip(sd, sh):
            if sm_d is not None:
                for a, b in zip(sm_d, sm_h):
                    assert a["iterations"] == b["iterations"], step
            for (xd, smd, vd, rhod, nxd), (xh, smh, vh, rhoh, nxh) in zip(rd, rh):
                assert smd["iterations"] == smh["iterations"], step
                vd, vh = np.asarray(vd, dtype=bool), np.asarray(vh, dtype=bool)
                assert np.array_equal(vd, vh), step
                worst = max(worst, np.abs(xd - xh).max())
                assert np.abs(xd - xh).max() < SEQ_TOL, step
                if len(rhod):
                    assert np.allclose(rhod[vd], rhoh[vh], rtol=SEQ_TOL, atol=0), step
                    assert np.allclose(nxd[vd], nxh[vh], rtol=SEQ_TOL, atol=0), step
        replaced += nonkey
        fd = paths[0].p.bw.download(paths[0].p.slots, 400)
        fh = paths[1].p.bw.download(paths[1].p.slots, 400)
        for a, b in zip(fd, fh):
            assert np.array_equal(a["ids"], b["ids"])
            worst = max(worst, np.abs(a["frames"] - b["frames"]).max())
            assert np.abs(a["frames"] - b["frames"]).max() < SEQ_TOL, step
            ok = a["n_obs"] > 0
            assert np.allclose(a["inv_depth"][ok], b["inv_depth"][ok], rtol=SEQ_TOL, atol=0), step
    assert replaced >= 5 and anchored_next > 20
    print(f"largest state difference between the two paths: {worst:.3e}; {anchored_next} tracks entered at a "
          f"replacing frame with inv_depth_next")
    ba.close()
