"""Phase times of marg_eig_kernel (tuning build with -DPVIO_MARG_STAMPS):
    python -c "from pvio_b200 import build as b; b.build(defines=['PVIO_MARG_STAMPS'], out='tools/_variants/libpvio_margstamps.so')"
    PVIO_B200_TUNE_LIB=$PWD/tools/_variants/libpvio_margstamps.so python tools/marg_stamps.py"""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from synthetic import synth
from pvio_b200 import _lib
from pvio_b200.bundle_adjustor import BundleAdjustor
w, s, _ = synth.make_cfg3()
b = BundleAdjustor(max_windows=1, max_frames=9, max_landmarks=320, max_obs=2560)
for _ in range(3):
    b.marginalize_frame(w, s, 0)
t = time.perf_counter()
for _ in range(10):
    b.marginalize_frame(w, s, 0)
print("marginalize_frame call ms", (time.perf_counter() - t) * 100)
st = np.zeros(8, dtype=np.int64)
assert b.lib.pvio_b200_debug_marg_stamps(_lib.ptr(st)) == 0
for n, v in zip(["tred2 (Householder tridiagonalisation)", "accumulate the transformations", "tql2 (implicit QL + eigenvectors)", "S, e"], np.diff(st[:5])):
    print(f"   {n:42s} {int(v):9d} cycles  {v / 1.965e3:8.1f} us")
b.close()
