"""The ctypes record of pvio_b200_batch_window_set_imu has the header's LP64 layout (no GPU needed)."""
import ctypes as C

from pvio_b200 import _lib


def test_imu_record_matches_the_header():
    R = _lib.CWindowImu
    assert C.sizeof(R) == 40                                          # include/pvio_b200.h: 40 bytes on LP64
    assert (R.slot.offset, R.frame.offset, R.n_samples.offset) == (0, 4, 8)
    assert (R.samples.offset, R.t_end.offset, R.noise_cov.offset) == (16, 24, 32)
    for name in ("pvio_b200_batch_window_set_imu", "pvio_b200_batch_window_imu_records"):
        assert name in _lib.EXPORTS


def test_imu_record_layout_as_the_c_compiler_sees_it(tmp_path):
    """sizeof / offsetof from a C compile of the header itself"""
    import os
    import shutil
    import subprocess
    import pytest
    if shutil.which("gcc") is None:
        pytest.skip("gcc not installed")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "pvio_b200.h"\n'
                   'int main(void) { printf("%zu %zu %zu %zu %zu %zu %zu\\n", sizeof(pvio_b200_window_imu),'
                   ' offsetof(pvio_b200_window_imu, slot), offsetof(pvio_b200_window_imu, frame),'
                   ' offsetof(pvio_b200_window_imu, n_samples), offsetof(pvio_b200_window_imu, samples),'
                   ' offsetof(pvio_b200_window_imu, t_end), offsetof(pvio_b200_window_imu, noise_cov)); return 0; }\n')
    exe = tmp_path / "layout"
    r = subprocess.run(["gcc", "-std=c99", "-I", os.path.join(root, "include"), str(src), "-o", str(exe)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True).stdout.split()]
    R = _lib.CWindowImu
    assert got == [C.sizeof(R), R.slot.offset, R.frame.offset, R.n_samples.offset, R.samples.offset, R.t_end.offset,
                   R.noise_cov.offset]
