"""Phase times of solve_kernel on the cfg3 / cfg4 / cfg2 single window (tuning build with -DPVIO_SOLVE_STAMPS):
    python -c "from pvio_b200 import build as b; b.build(defines=['PVIO_SOLVE_STAMPS'], out='tools/_variants/libpvio_stamps.so')"
    PVIO_B200_TUNE_LIB=$PWD/tools/_variants/libpvio_stamps.so python tools/solve_stamps.py"""
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from synthetic import synth
from pvio_b200 import _lib
from pvio_b200.bundle_adjustor import BundleAdjustor

NAMES = ["init+T", "vision blocks", "imu_factor_raw", "imu whiten+accumulate", "prior r, S^T r", "prior H, g", "planes",
         "scale / mask", "cholesky + solve", "outputs"]
for name, maker in (("cfg3", synth.make_cfg3), ("cfg4", synth.make_cfg4), ("cfg2", synth.make_cfg2)):
    w, s, _ = maker()
    ba = BundleAdjustor(max_windows=1, max_frames=10, max_landmarks=512, max_obs=4608)
    for _ in range(3):
        ba.gn_step(w, s)
    st = np.zeros(16, dtype=np.int64)
    assert ba.lib.pvio_b200_debug_solve_stamps(_lib.ptr(st)) == 0
    d = np.diff(st[:10])
    print(name, "total cycles", int(st[9] - st[0]), "=", round((st[9] - st[0]) / 1.965e3, 1), "us at 1.965 GHz")
    for n, v in zip(NAMES[1:], d):
        if abs(v) < 1e8:
            print(f"   {n:26s} {int(v):8d} cycles  {v / 1.965e3:7.1f} us")
    print("   cholesky, summed over block columns: thread 0 (diagonal warp): wait for the panel", st[10], "diag update + factor + rest", st[11],
          "| thread 32: panel", st[12], "barrier", st[13], "trailing", st[14], "barrier", st[15])
    ba.close()
