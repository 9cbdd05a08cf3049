"""SlidingWindowTracker::mirror_frame (pvio/src/pvio/core/sliding_window_tracker.cpp:52-73) restated over keypoint
lists, and the frame edit that pvio_b200_batch_window_mirror_frame derives from it.

Frame i is the window's newest frame, frame j the tracker's new frame.  `prev_index` [n_j] is batch_feature_track's:
the keypoint of frame i each keypoint of frame j continues, or -1; `track_of` {ki: track id} maps frame i's keypoints
to the window's tracks.  Two orders come out of the mirror:
  - the list order (kj ascending): PnP residual blocks and the parallax list walk frame j's keypoints
    (pnp.cpp:56, sliding_window_tracker.cpp:269);
  - the id order (ki ascending): mirror_frame creates a track for a keypoint of frame i without one while it walks
    frame i (:66-71), so the window's next ids go to the valid candidates in ki order."""


def mirror_frame(prev_index, track_of):
    """(continued, candidates): continued [(kj, track id)] in kj order; candidates [(ki, kj)] in ki order, the
    keypoints of frame i without a track that frame j continues"""
    kj_of = {int(ki): kj for kj, ki in enumerate(prev_index) if ki >= 0}
    continued = [(kj, track_of[int(ki)]) for kj, ki in enumerate(prev_index) if ki >= 0 and int(ki) in track_of]
    candidates = [(ki, kj_of[ki]) for ki in sorted(kj_of) if ki not in track_of]
    return continued, candidates


def pnp_list(continued, role, given):
    """the PnP observations [(kj, track id)] in kj order: a landmark (role -1) always, a track of role -2 or a plane
    index only with a given point (a TF_PLANE track takes its plane-cast point, pnp.cpp:62-85)"""
    return [(kj, t) for kj, t in continued if role.get(t, -1) == -1 or t in given]


def parallax_pairs(continued, candidates, frames_of, frame_i, newest):
    """the keyframe check's pairs: every continued track with a keypoint in frame_i ([(kj, track id)], kj order), and
    every candidate when frame_i is the newest frame (keyframe_check walks every track of frame j, :269-277)"""
    pairs = [(kj, t) for kj, t in continued if frame_i in frames_of[t]]
    return pairs, (list(candidates) if frame_i == newest else [])


def append(continued, candidates, valid, next_id, replace, ends):
    """kp_track {kj: track id} after the frame edit and the slot's next id: the continued tracks, except those that
    `ends` (observed in the replaced frame only) when the newest frame is replaced, and the valid candidates with the
    next ids in ki order"""
    kp = {kj: t for kj, t in continued if not (replace and t in ends)}
    k = 0
    for (ki, kj), v in zip(candidates, valid):
        if v:
            kp[kj] = next_id + k
            k += 1
    return kp, next_id + k
