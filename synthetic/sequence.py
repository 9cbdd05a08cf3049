"""Sliding-window SEQUENCE on top of one long synthetic run (test harness: plays the role of PVIO's
SlidingWindowTracker / Map bookkeeping, core/sliding_window_tracker.cpp:75-125, map/map.cpp:76-88, map/track.cpp:42-49).

A run of F keyframes (synth.make_cfg3 with N = F: trajectory, landmarks with their track frames, one IMU factor per
consecutive pair) is cut into windows of N frames.  Per keyframe the caller (a) solves the window, (b) marginalises its
oldest frame into a prior over the remaining N - 1 frames, (c) shifts: drops the oldest frame, appends the next one.
`Chain` carries one estimator's state along the run (frame states, inverse depths with their anchors, the prior), so a
GPU chain and an oracle chain can be advanced side by side with their own numbers."""
import dataclasses

import numpy as np

from pvio_b200.window import Window, State
from . import so3, synth


class Run:
    def __init__(self, F=26, N=6, M=260, seed=700, planes=0, tracks_per_plane=40, plane_landmarks=False):
        """planes > 0: synth.make_cfg3(planes=..., tracks_per_plane=...) over the long run; its plane tracks follow the
        landmarks in `tracks`.  plane_landmarks: those tracks stay ordinary landmarks (role -1) whose points lie on the
        known planes -- what a plane extractor finds before any track is a plane track -- drawn within 6 m and with
        0.05 px of keypoint noise, and the run starts from its true states, so that the solved points of those tracks
        stay within the extractor's 3 cm of the plane"""
        self.F, self.N, self.plane_landmarks = F, N, plane_landmarks
        self.w, self.guess, self.truth = synth.make_cfg3(seed=seed, N=F, M=M, prior='none', planes=planes,
                                                         tracks_per_plane=tracks_per_plane,
                                                         plane_noise_px=0.05 if plane_landmarks else None,
                                                         plane_range=(1.0, 6.0) if plane_landmarks else (1.0, 15.0))
        if plane_landmarks:
            self.guess = self.truth.copy()
        w = self.w
        self.tracks = []                      # per track (landmarks, then plane tracks): sorted frame list and keypoints
        for l in range(w.M):
            fr = [int(w.lm_anchor[l])] + [int(f) for f in w.obs_frame[w.lm_obs_begin[l]:w.lm_obs_begin[l + 1]]]
            zs = [w.lm_z_ref[l]] + [w.obs_z[k] for k in range(w.lm_obs_begin[l], w.lm_obs_begin[l + 1])]
            self.tracks.append((fr, zs))
        self.plane_of = [-1] * w.M            # per track: the plane a plane track was drawn on, -1 for a landmark
        self.rho0 = list(self.guess.rho)      # per track: initial inverse depth in its first frame
        for t in range(w.n_ptracks):          # plane points: the anchor ray meets the plane (guess pose of the anchor)
            ks = range(int(w.pt_obs_begin[t]), int(w.pt_obs_begin[t + 1]))
            fr, zs = [int(w.pt_obs_frame[k]) for k in ks], [w.pt_obs_z[k] for k in ks]
            self.tracks.append((fr, zs))
            p = int(w.pt_plane[t])
            self.plane_of.append(p)
            qc, pc = self.cam_pose(self.guess.q[fr[0]], self.guess.p[fr[0]])
            u = so3.qrot(qc, np.array([zs[0][0], zs[0][1], 1.0]))
            self.rho0.append((w.plane_normal[p] @ u) / (w.plane_distance[p] - w.plane_normal[p] @ pc))
        self.rho0 = np.array(self.rho0)

    def role(self, l, k):
        """The role the host shim gives track l in the window of keyframe k (pvio_b200_window_planes): the plane
        extractor casts every 11th landmark onto a plane from keyframe 3; every 7th plane track is revalidated off its
        plane at keyframe 5 and stays a landmark; plane 1 has fewer than 20 tracks in keyframes 4 .. 7 (role -2).  With
        plane_landmarks every track is a landmark."""
        n_planes, p = self.w.n_planes, self.plane_of[l]
        if self.plane_landmarks:
            return -1
        if p < 0:
            return (l // 11) % n_planes if n_planes > 0 and l % 11 == 0 and k >= 3 else -1
        if (l - self.w.M) % 7 == 0 and k >= 5:
            return -1
        return -2 if p == 1 and 4 <= k < 8 else p

    def planes_at(self, k):
        """[n_planes][4] the plane parameters of keyframe k (the extractor refines them after every keyframe)"""
        w = self.w
        return np.concatenate([w.plane_normal, (w.plane_distance + 1e-3 * k)[:, None]], axis=1)

    def revalidated_rho(self, l):
        """the inverse depth the revalidation gives a plane track that becomes a landmark (set_landmark_point), in its
        anchor frame at that keyframe"""
        return 1.1 * self.rho0[l]

    def cam_pose(self, q, p):
        return so3.qmul(q, self.w.cam_q_cs), p + so3.qrot(q, self.w.cam_p_cs)


class Chain:
    """One estimator's view of the run: absolute frame states [F], per-landmark (anchor frame, inverse depth), prior."""

    def __init__(self, run):
        self.run = run
        g = run.guess
        self.q, self.p, self.v, self.bg, self.ba = g.q.copy(), g.p.copy(), g.v.copy(), g.bg.copy(), g.ba.copy()
        self.anchor = np.array([t[0][0] for t in run.tracks])
        self.rho = run.rho0.copy()
        self.prior = None                     # dict(frames (absolute), S, e, x0 [n][16])
        self.roles = {}                       # track -> role in the last gathered window (tracks seen there)
        self.pt_ids = []                      # plane tracks of the last gathered window, in the order of its pt tables

    def _reanchor(self, l, new_anchor):
        """Track::first_frame changes when the old anchor leaves the window: the inverse depth is re-expressed in the next
        observing frame from the CURRENT estimate (map/track.cpp:42-49)."""
        run = self.run
        fr, zs = run.tracks[l]
        a = int(self.anchor[l])
        qc, pc = run.cam_pose(self.q[a], self.p[a])
        z = zs[fr.index(a)]
        x = so3.qrot(qc, np.array([z[0], z[1], 1.0]) / self.rho[l]) + pc
        qn, pn = run.cam_pose(self.q[new_anchor], self.p[new_anchor])
        y = so3.qrot(so3.qconj(qn), x - pn)
        self.anchor[l] = new_anchor
        self.rho[l] = 1.0 / y[2]

    def window(self, k):
        """Window over absolute frames [k, k + N): (Window, State, landmark ids).  With planes (Run.role): landmarks are
        the tracks of role < 0 with >= 2 observations (role -2: lm_in_victim = 0), plane tracks those of role >= 0 with all
        their observations, in the order the resident slot creates them (first frame, then track); a plane track that
        becomes a landmark takes Run.revalidated_rho."""
        run, N = self.run, self.run.N
        src = run.w
        w = dataclasses.replace(src)
        w.N = N
        w.frame_fixed = np.zeros(N, dtype=np.uint8)
        lm_ids, anchors, zref, begins, of, oz, victim, rho = [], [], [], [0], [], [], [], []
        pts = []
        for l, (fr, zs) in enumerate(run.tracks):
            inw = [(f, z) for f, z in zip(fr, zs) if k <= f < k + N]
            if not inw:
                continue
            role, prev = run.role(l, k), self.roles.get(l, -1)
            self.roles[l] = role
            if len(inw) < 2 and role < 0:
                continue
            if self.anchor[l] != inw[0][0]:
                if self.anchor[l] < inw[0][0]:
                    self._reanchor(l, inw[0][0])
                else:
                    continue
            if prev >= 0 and role == -1:
                self.rho[l] = run.revalidated_rho(l)
            if role >= 0:
                pts.append((fr[0], l, role, inw))
                continue
            lm_ids.append(l)
            anchors.append(inw[0][0] - k)
            zref.append(inw[0][1])
            for f, z in inw[1:]:
                of.append(f - k)
                oz.append(z)
            begins.append(len(of))
            victim.append(1 if inw[0][0] == k and role != -2 else 0)
            rho.append(self.rho[l])
        w.M, w.K = len(lm_ids), len(of)
        w.lm_anchor = np.array(anchors, dtype=np.int32)
        w.lm_z_ref = np.array(zref).reshape(-1, 2)
        w.lm_obs_begin = np.array(begins, dtype=np.int32)
        w.obs_frame = np.array(of, dtype=np.int32)
        w.obs_z = np.array(oz).reshape(-1, 2)
        w.lm_in_victim = np.array(victim, dtype=np.uint8)
        sl = slice(k, k + N - 1)
        w.n_imu = N - 1
        w.imu_frame_i = np.arange(0, N - 1, dtype=np.int32)
        w.imu_frame_j = np.arange(1, N, dtype=np.int32)
        for name in ('imu_dt', 'imu_dq', 'imu_dp', 'imu_dv', 'imu_sqrt_inv_cov', 'imu_dq_dbg', 'imu_dp_dbg', 'imu_dp_dba',
                     'imu_dv_dbg', 'imu_dv_dba', 'imu_bg0', 'imu_ba0'):
            setattr(w, name, getattr(src, name)[sl].copy())
        st = State(self.q[k:k + N].copy(), self.p[k:k + N].copy(), self.v[k:k + N].copy(), self.bg[k:k + N].copy(),
                   self.ba[k:k + N].copy(), np.array(rho))
        if self.prior is None:
            synth.gauge_prior(w, st)          # first window: 1e15 on the pose of frame 0 (sliding_window_tracker.cpp:100-112)
        else:
            pr = self.prior
            w.n_prior = len(pr['frames'])
            w.prior_frames = (np.array(pr['frames']) - k).astype(np.int32)
            w.prior_S, w.prior_e = pr['S'], pr['e']
            x0 = pr['x0']
            w.prior_q0, w.prior_p0, w.prior_v0 = x0[:, 0:4].copy(), x0[:, 4:7].copy(), x0[:, 7:10].copy()
            w.prior_bg0, w.prior_ba0 = x0[:, 10:13].copy(), x0[:, 13:16].copy()
        pts.sort(key=lambda t: t[:2])
        self.pt_ids = [t[1] for t in pts]
        w.n_planes = src.n_planes
        if src.n_planes > 0:
            pl = run.planes_at(k)
            w.plane_normal, w.plane_distance = pl[:, :3].copy(), pl[:, 3].copy()
        w.n_ptracks = len(pts)
        w.pt_plane = np.array([t[2] for t in pts], dtype=np.int32)
        w.pt_obs_begin = np.concatenate([[0], np.cumsum([len(t[3]) for t in pts])]).astype(np.int32)
        w.pt_obs_frame = np.array([f - k for t in pts for f, _ in t[3]], dtype=np.int32)
        w.pt_obs_z = np.array([z for t in pts for _, z in t[3]]).reshape(-1, 2)
        w.validate()
        return w, st, lm_ids

    def store(self, k, st, lm_ids):
        N = self.run.N
        self.q[k:k + N], self.p[k:k + N], self.v[k:k + N] = st.q, st.p, st.v
        self.bg[k:k + N], self.ba[k:k + N] = st.bg, st.ba
        for i, l in enumerate(lm_ids):
            self.rho[l] = st.rho[i]

    def set_prior(self, k, S, e, st):
        """The prior produced by marginalising frame k: over absolute frames k + 1 .. k + N - 1, linearised at st."""
        N = self.run.N
        x0 = np.concatenate([st.q[1:], st.p[1:], st.v[1:], st.bg[1:], st.ba[1:]], axis=1)
        self.prior = dict(frames=list(range(k + 1, k + N)), S=S, e=e, x0=x0)


class ResidentPlayer:
    """Feeds a run into the RESIDENT window of a handle (pvio_b200.resident.ResidentWindow): what the shim does with the
    resident API -- per keyframe: solve, drop the victim, append the next frame with its observations."""

    def __init__(self, ba, run):
        from pvio_b200 import _lib
        from pvio_b200.resident import ResidentWindow
        self.run, self.rw, self.ids = run, ResidentWindow(ba, run.w), {}
        g = run.guess
        self.rec = _lib.PackedArgs(run.w, g).keep["imu"].reshape(-1, 288)     # factor f couples absolute frames (f, f + 1)
        for f in range(run.N):
            self.rw.append_frame(self.state16(f), False, self.rec[f - 1] if f > 0 else None)
            self.feed(f, f)
        w0, _, _ = Chain(run).window(0)                                       # first window: the 1e15 gauge prior
        x0 = np.concatenate([w0.prior_q0, w0.prior_p0, w0.prior_v0, w0.prior_bg0, w0.prior_ba0], axis=1)
        self.rw.set_prior(w0.prior_S, w0.prior_e, x0)
        self.seconds = 0.0                                                    # wall time spent inside the C-ABI calls

    def state16(self, f):
        g = self.run.guess
        return np.concatenate([g.q[f], g.p[f], g.v[f], g.bg[f], g.ba[f]])

    def feed(self, f_abs, f_win):
        new, seen = [], []
        for l, (fr, zs) in enumerate(self.run.tracks):
            if f_abs in fr:
                (seen if l in self.ids else new).append((l, zs[fr.index(f_abs)]))
        if seen:
            self.rw.add_observations([self.ids[l] for l, _ in seen], [f_win] * len(seen), [z for _, z in seen])
        if new:
            got = self.rw.add_tracks([f_win] * len(new), [z for _, z in new], [self.run.guess.rho[l] for l, _ in new])
            for (l, _), i in zip(new, got):
                self.ids[l] = int(i)

    def solve(self, max_iterations):
        import time
        t = time.perf_counter()
        s = self.rw.solve(max_iterations=max_iterations)
        self.seconds += time.perf_counter() - t
        return s

    def shift(self, k):
        """drop frame k (the oldest), append absolute frame k + N"""
        import time
        f_abs = k + self.run.N
        t = time.perf_counter()
        self.rw.drop_victim()
        self.rw.append_frame(self.state16(f_abs), False, self.rec[f_abs - 1])
        self.seconds += time.perf_counter() - t
        self.feed(f_abs, self.run.N - 1)


class WindowModel:
    """Host model of one resident slot, as the map sees it: absolute frames in the window and, per live track, its
    landmark, window frames (increasing), keypoints and inverse depth.  It applies the same edits and drops as
    pvio_b200_batch_window_* (erase_frame / put_frame / add_keypoint / prune_tracks / marginalize_frame(0) of
    map/map.cpp, without the re-anchoring, which needs states), and gives the window a gather would pack."""

    def __init__(self):
        self.frames, self.tracks, self.next_id = [], {}, 0

    def edit(self, e, f_abs=None):
        """apply an Edit; f_abs: the absolute id of its new frame.  Returns the new track ids."""
        if e.replace_last:                                   # map->erase_frame(frame_num - 1)
            last = len(self.frames) - 1
            self.frames.pop()
            for i in list(self.tracks):
                t = self.tracks[i]
                if t['frames'][-1] == last:
                    t['frames'].pop(); t['zs'].pop()
                if not t['frames']:
                    del self.tracks[i]
        if e.state is not None:
            self.frames.append(f_abs)
        ids = []
        for (f, z, rho), l in zip(e.new, getattr(e, 'landmarks', [None] * len(e.new))):
            self.tracks[self.next_id] = dict(l=l, frames=[f], zs=[np.asarray(z, dtype=float)], rho=rho, role=-1)
            ids.append(self.next_id)
            self.next_id += 1
        for i, f, z in e.obs:
            if i in self.tracks:
                self.tracks[i]['frames'].append(f); self.tracks[i]['zs'].append(np.asarray(z, dtype=float))
        for i in e.remove:
            del self.tracks[i]
        return ids

    def drop(self):
        """marginalize_frame(0): the victim's keypoints leave their tracks, indices shift"""
        self.frames.pop(0)
        for i in list(self.tracks):
            t = self.tracks[i]
            if t['frames'][0] == 0:
                t['frames'].pop(0); t['zs'].pop(0)
            if not t['frames']:
                del self.tracks[i]
                continue
            t['frames'] = [f - 1 for f in t['frames']]

    def set_planes(self, p):
        """apply a pvio_b200.batch_window.Planes record: the roles of its tracks"""
        for i, role in zip(p.tracks, p.roles):
            self.tracks[i]['role'] = role

    def view(self):
        """landmark -> (anchor, z_ref, obs frames, obs keypoints) of the tracks of role < 0 with >= 2 observations, in
        id order"""
        out = {}
        for i in sorted(self.tracks):
            t = self.tracks[i]
            if t['role'] < 0 and len(t['frames']) >= 2:
                out[t['l']] = (t['frames'][0], t['zs'][0], list(t['frames'][1:]), [z for z in t['zs'][1:]])
        return out

    def victims(self):
        """landmark -> lm_in_victim of the landmarks of view(): anchored in frame 0 and not role -2"""
        return {t['l']: int(t['frames'][0] == 0 and t['role'] != -2) for t in self.tracks.values()
                if t['role'] < 0 and len(t['frames']) >= 2}

    def plane_view(self):
        """the plane tracks (role >= 0) in id order: (landmark, plane, frames, keypoints)"""
        return [(t['l'], t['role'], list(t['frames']), list(t['zs']))
                for t in (self.tracks[i] for i in sorted(self.tracks)) if t['role'] >= 0]


class ModelWindows:
    """The host models of several slots behind the interface of pvio_b200.batch_window.BatchWindows (edits, drops, the
    live ids of a download): a BatchPlayer runs on it without a device."""

    def __init__(self):
        self.m = {}

    def reset(self, slot, win):
        self.m[slot] = WindowModel()

    def set_prior(self, slot, S, e, x0):
        pass

    def edit(self, edits):
        return [np.array(self.m[e.slot].edit(e, getattr(e, 'f_abs', None)), dtype=np.int32) for e in edits]

    def set_planes(self, records):
        for p in records:
            self.m[p.slot].set_planes(p)

    def set_imu(self, records):
        pass

    def drop_victim(self, slots, want=False):
        for s in slots:
            self.m[s].drop()

    def download(self, slots, track_stride):
        return [dict(ids=np.array(sorted(self.m[s].tracks), dtype=np.int32)) for s in slots]


class BatchPlayer:
    """Feeds several runs into RESIDENT batched slots (pvio_b200.batch_window.BatchWindows): run j lives in slot
    slots[j].  Per keyframe of a slot: solve, drop the victim, then the next camera frame arrives first as a non-keyframe
    (a perturbed state with the frame's observations) that the real keyframe replaces (replace_last), as PVIO's tracker
    erases a non-keyframe newest frame (sliding_window_tracker.cpp:115-121).  The host model keeps, per slot, the live
    track of each landmark (`ids`) and the window's first absolute frame (`k`).
    With imu_samples, every frame edit with an IMU factor is followed by a set_imu with the factor's raw samples
    (Run.truth.imu_factors), so the slots re-integrate their factors before each solve; off, the factors keep the
    records of their edits (integrated once, at the guess biases)."""

    def __init__(self, ba, runs, slots=None, bw=None, imu_samples=False):
        """ba: the handle's BundleAdjustor; bw (instead of ba): any object with BatchWindows' interface (ModelWindows).
        `model` (a ModelWindows) follows every edit and drop: the window a gather of the map would pack."""
        from pvio_b200 import _lib
        from pvio_b200.batch_window import BatchWindows, Edit, Imu, Planes
        self.Edit, self.Planes, self.Imu, self.imu_samples = Edit, Planes, Imu, imu_samples
        self.runs, self.bw = runs, (BatchWindows(ba) if bw is None else bw)
        self.model = bw if isinstance(bw, ModelWindows) else ModelWindows()
        self.slots = list(range(len(runs))) if slots is None else list(slots)
        self.ids = [dict() for _ in runs]                  # landmark -> live track id
        self.roles = [dict() for _ in runs]                # landmark -> role of its live track
        self.k = [0] * len(runs)
        self.rec = [_lib.PackedArgs(r.w, r.guess).keep["imu"].reshape(-1, 288) for r in runs]
        for j, r in enumerate(runs):
            self.bw.reset(self.slots[j], r.w)
            if self.model is not self.bw:
                self.model.reset(self.slots[j], r.w)
        for f in range(max(r.N for r in runs)):
            js = [j for j, r in enumerate(runs) if f < r.N]
            self._apply([self.frame_edit(j, f, f) for j in js], js)
        for j, r in enumerate(runs):
            w0, _, _ = Chain(r).window(0)                   # first window: the 1e15 gauge prior
            x0 = np.concatenate([w0.prior_q0, w0.prior_p0, w0.prior_v0, w0.prior_bg0, w0.prior_ba0], axis=1)
            self.bw.set_prior(self.slots[j], w0.prior_S, w0.prior_e, x0)
        self.set_roles(list(range(len(runs))))

    def state16(self, j, f):
        g = self.runs[j].guess
        return np.concatenate([g.q[f], g.p[f], g.v[f], g.bg[f], g.ba[f]])

    def frame_edit(self, j, f_abs, f_win, replace_last=False, state=None):
        """the edit that appends absolute frame f_abs at window index f_win, with its observations and new tracks"""
        r = self.runs[j]
        e = self.Edit(self.slots[j], replace_last).frame(self.state16(j, f_abs) if state is None else state, False,
                                                         self.rec[j][f_abs - 1] if f_abs > 0 and f_win > 0 else None)
        e.landmarks, e.f_abs, e.f_win = [], f_abs, f_win
        for l, (fr, zs) in enumerate(r.tracks):
            if f_abs in fr:
                z = zs[fr.index(f_abs)]
                if l in self.ids[j]:
                    e.obs.append((self.ids[j][l], f_win, z))
                else:
                    e.new.append((f_win, z, r.rho0[l]))
                    e.landmarks.append(l)
        return e

    def imu(self, j, f_win, f_abs, first=None):
        """the Imu record of window frame f_win = absolute frame f_abs of run j: the raw samples of the factors from
        absolute frame `first` (default f_abs - 1) to f_abs back to back -- a frame that replaces an erased
        non-keyframe holds the merged list (sliding_window_tracker.cpp:116-117)"""
        fs = self.runs[j].truth.imu_factors
        first = f_abs - 1 if first is None else first
        smp = np.concatenate([fs[g][0] for g in range(first, f_abs)])
        return self.Imu(self.slots[j], f_win, smp, fs[f_abs - 1][1], self.runs[j].truth.imu_noise)

    def _apply(self, edits, js):
        got = self.bw.edit(edits)
        if self.model is not self.bw:
            self.model.edit(edits)
        if self.imu_samples:
            recs = [self.imu(j, e.f_win, e.f_abs) for e, j in zip(edits, js) if e.imu is not None]
            if recs:
                self.bw.set_imu(recs)
        for e, j, ids in zip(edits, js, got):
            for l, i in zip(e.landmarks, ids):
                self.ids[j][l] = int(i)
                self.roles[j][l] = -1

    def set_roles(self, js):
        """the roles of keyframe self.k[j] (Run.role) and the plane parameters of the runs js with planes, in one
        set_planes: a changed role per live track, and a plane track that becomes a landmark with its new inverse depth"""
        recs = []
        for j in js:
            r = self.runs[j]
            if r.w.n_planes == 0:
                continue
            k, p = self.k[j], self.Planes(self.slots[j], r.planes_at(self.k[j]))
            for l, i in sorted(self.ids[j].items(), key=lambda t: t[1]):
                old, new = self.roles[j].get(l, -1), r.role(l, k)
                if new != old:
                    p.role(i, new, r.revalidated_rho(l) if old >= 0 and new == -1 else np.nan)
                    self.roles[j][l] = new
            recs.append(p)
        if recs:
            self.bw.set_planes(recs)
            if self.model is not self.bw:
                self.model.set_planes(recs)

    def refresh(self, js, track_stride):
        """download the slots of runs js; forget the landmarks whose tracks died"""
        out = self.bw.download([self.slots[j] for j in js], track_stride)
        for j, d in zip(js, out):
            live = set(int(i) for i in d["ids"])
            self.ids[j] = {l: i for l, i in self.ids[j].items() if i in live}
        return out

    def advance(self, js, perturb=1e-3, nonkey=True):
        """drop the victim of the runs js, then their next frame -- first as a non-keyframe that the keyframe replaces
        (nonkey), or directly"""
        self.bw.drop_victim([self.slots[j] for j in js])
        if self.model is not self.bw:
            self.model.drop_victim([self.slots[j] for j in js])
        self.refresh(js, max(len(r.tracks) for r in self.runs))
        for j in js:
            self.k[j] += 1
        if not nonkey:
            self._apply([self.frame_edit(j, self.k[j] + self.runs[j].N - 1, self.runs[j].N - 1) for j in js], js)
            self.set_roles(js)
            return
        fake = []
        for j in js:
            f_abs, N = self.k[j] + self.runs[j].N - 1, self.runs[j].N
            s = self.state16(j, f_abs).copy()
            s[4:7] += perturb
            fake.append(self.frame_edit(j, f_abs, N - 1, state=s))
        self._apply(fake, js)
        for e, j in zip(fake, js):                          # the non-keyframe's new tracks die with it
            for l in e.landmarks:
                del self.ids[j][l]
        real = [self.frame_edit(j, self.k[j] + self.runs[j].N - 1, self.runs[j].N - 1, replace_last=True) for j in js]
        self._apply(real, js)
        self.set_roles(js)
