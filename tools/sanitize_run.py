"""Small end-to-end pass over every kernel for compute-sanitizer (memcheck / racecheck / initcheck)."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from pvio_b200 import klt
from synthetic import synth
from pvio_b200.bundle_adjustor import BundleAdjustor
ba = BundleAdjustor(max_windows=80, max_frames=8, max_landmarks=96, max_obs=800)
w, st, _ = synth.make_cfg2(N=6, M=70, staggered=True)
print('gn_step cfg2', np.linalg.norm(ba.gn_step(w, st)['dx']))
for i in range(80):
    ba.batch_set(i, w, st)
ba.batch_upload(80); ba.batch_gn_step(80, 1e-8, apply=True); dx, c = ba.batch_download(80, 15 * 6 + 70)
print('batch 80 (one CTA per window + lean solve)', np.linalg.norm(dx[79]), c[0])
w3, st3, _ = synth.make_cfg3(N=6, M=60)
print('gn_step cfg3', np.linalg.norm(ba.gn_step(w3, st3)['dx']))
w4, st4, _ = synth.make_cfg4(N=6, M=40, tracks_per_plane=20)
print('gn_step cfg4', np.linalg.norm(ba.gn_step(w4, st4)['dx']))
s, summ = ba.solve(w3, st3, max_iterations=3)
print('solve', summ['iterations'], summ['final_cost'])
S, e = ba.marginalize_frame(w3, st3, 0)
print('marg', np.linalg.norm(S), np.linalg.norm(e))
print('reproj err', ba.compute_reprojection_error(w, st))
prev, nxt, pts, _ = synth.make_klt_pair(size=(160, 120), n_points=20)
p, s_, e_ = klt.track_keypoints(ba, prev, nxt, pts)
print('klt', int(s_.sum()))
# LK windows folding at a 22-px level (176 x 176, level 3) and on a frame narrower than the window, points beyond the edge
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests'))
from test_klt_oracle_edges import edge_case
for size in ((176, 176), (12, 12)):
    ep, en, epts, einit, _ = edge_case(size)
    print('klt edges', size, int(klt.track_keypoints(ba, ep, en, epts, einit, raw=True)[1].sum()))
# PnP, IMU pre-integration, triangulation, Lie self-test, batched device-side solve
from pvio_b200 import pnp, imu, triangulate as tri
d = synth.make_pnp()
_, ps = pnp.visual_inertial_pnp(ba, d['frame'], d['last'], d['imu'], d['pts'], d['zs'], d['cam_q'], d['cam_p'], d['imu_q'], d['imu_p'], d['W'], True)
print('pnp', ps['iterations'])
_, _, truth = synth.make_cfg3(N=4, M=30)
print('imu', np.linalg.norm(imu.preintegrate(ba, truth.imu_factors, truth.imu_noise)[:, :11]))
P = np.array([np.c_[np.eye(3), -np.array([0.3 * i, 0, 0])] for i in range(4)])      # identity rotation, camera at (0.3 i, 0, 0)
X = np.array([0.2, 0.1, 5.0])
zz = np.array([(P[f] @ np.r_[X, 1])[:2] / (P[f] @ np.r_[X, 1])[2] for f in range(4)])
print('tri', tri.triangulate(ba, P, [0, 4], [0, 1, 2, 3], zz)[0])
print('lie', np.linalg.norm(ba.selftest_lie(np.array([[0.1, 0.2, 0.3], [1e-9, 0, 0], [3.14159, 0, 0]]))))
ba.batch_set(0, w, st); ba.batch_replicate(80); ba.batch_upload(80); ba.batch_solve(80, max_iterations=3)
fr, rh, sm = ba.batch_download_state(80, w.N, w.M)
print('batch solve', sm[0]['iterations'], sm[79]['final_cost'])
ba.close()
# round 2: F-matrix RANSAC (+ LMedS branch, whole track_keypoints), detector, the 135-dim inertial window (register-resident
# Cholesky, 5-slot instantiation at N = 11), the failure / retry path, the producer / consumer eigen-solver at D = 135
from pvio_b200.detect import detect_keypoints
b2 = BundleAdjustor(max_windows=1, max_frames=12, max_landmarks=512, max_obs=4608)
fp, fq = synth.make_fm_matches(5, 200, 0.3)
m, F, info = klt.find_fundamental_mask(b2, fp, fq, return_info=True)
print('fm ransac', int(m.sum()), info)
m, F, info = klt.find_fundamental_mask(b2, fp[:14], fq[:14], return_info=True)
print('fm lmeds', int(m.sum()), info)
nx, stt = klt.track_keypoints_ransac(b2, prev, nxt, pts, prev_id=11, next_id=12)
print('track_keypoints whole', int(stt.sum()))
kp = detect_keypoints(b2, nxt, pts[:5], keypoint_distance=15.0, clahe_clip=6.0, frame_id=12)
print('detect', len(kp))
for N in (9, 11):
    wN, sN, _ = synth.make_cfg3(N=N, M=120)
    o, sm_ = b2.solve(wN, sN, max_iterations=3)
    print('solve cfg3 N', N, sm_['iterations'], sm_['final_cost'])
    S, e = b2.marginalize_frame(wN, sN, 0)
    print('marg N', N, np.linalg.norm(S))
w4b, s4b, _ = synth.make_cfg4(N=9, M=100)
o, sm_ = b2.solve(w4b, s4b, max_iterations=2)
print('solve cfg4', sm_['iterations'])
import copy
wb = copy.deepcopy(wN); wb.obs_z = wb.obs_z.copy(); wb.obs_z[3, 0] = np.nan
o, sm_ = b2.solve(wb, sN, max_iterations=10, postpass=False)
print('failure path', sm_['termination'], sm_['usable'])
b2.close()
