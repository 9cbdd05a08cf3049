"""The ctypes record of pvio_b200_batch_window_track_frame has the header's LP64 layout (no GPU needed)."""
import ctypes as C
import os
import shutil
import subprocess

import pytest

from pvio_b200 import _lib

FIELDS = ("slot", "newest_is_keyframe", "n_samples", "n_merge", "samples", "merge_samples", "t_end", "noise_cov", "cx",
          "cy", "skipped_frames", "state", "predicted", "imu_record", "keyframe", "parallax", "n_parallax", "n_obs",
          "obs_track", "obs_z", "obs_point", "points_out", "n_new", "new_z_last", "new_z", "new_valid", "new_inv_depth",
          "new_inv_depth_next", "summary")


def test_track_frame_record_matches_the_header():
    R = _lib.CWindowTrackFrame
    assert C.sizeof(R) == 216                                         # include/pvio_b200.h: 216 bytes on LP64
    assert [f for f, _ in R._fields_] == list(FIELDS)
    assert (R.slot.offset, R.n_merge.offset, R.samples.offset, R.t_end.offset, R.cx.offset) == (0, 12, 16, 32, 48)
    assert (R.skipped_frames.offset, R.keyframe.offset, R.n_obs.offset, R.n_new.offset, R.summary.offset) == (64, 96, 120, 160, 208)
    assert "pvio_b200_batch_window_track_frame" in _lib.EXPORTS


def test_track_frame_record_layout_as_the_c_compiler_sees_it(tmp_path):
    """sizeof / offsetof of every field from a C compile of the header itself"""
    if shutil.which("gcc") is None:
        pytest.skip("gcc not installed")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "layout.c"
    offs = "".join(f', offsetof(pvio_b200_window_track_frame, {f})' for f in FIELDS)
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "pvio_b200.h"\n'
                   'int main(void) { printf("' + "%zu " * (len(FIELDS) + 1) + '\\n", sizeof(pvio_b200_window_track_frame)'
                   + offs + '); return 0; }\n')
    exe = tmp_path / "layout"
    r = subprocess.run(["gcc", "-std=c99", "-I", os.path.join(root, "include"), str(src), "-o", str(exe)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True).stdout.split()]
    R = _lib.CWindowTrackFrame
    assert got == [C.sizeof(R)] + [getattr(R, f).offset for f in FIELDS]
