"""Writes tests/golden/lotbox3_golden.npz: the 3-draw sample schedules of PVIO's Ransac<3, ...> at seed 0, as the plane
RANSAC of PlaneExtractor::work and Plane::update_parameter draws them (utility/ransac.h), from the same small C++ program
as make_lotbox_golden.py, compiled here with g++ against <random> only.  Run: python tests/golden/make_lotbox3_golden.py"""
import os
import subprocess
import sys
import tempfile

import numpy as np

from make_lotbox_golden import ITERS, SRC

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = [(n, 0, 3) for n in (3, 4, 5, 31, 50, 300, 2000)]


def main():
    with tempfile.TemporaryDirectory() as tmp:
        src, exe = os.path.join(tmp, "lotbox.cpp"), os.path.join(tmp, "lotbox")
        with open(src, "w") as f:
            f.write(SRC)
        subprocess.run(["g++", "-std=c++17", "-O2", src, "-o", exe], check=True)
        out = {}
        for i, (n, seed, dof) in enumerate(CASES):
            r = subprocess.run([exe, str(n), str(seed), str(dof), str(ITERS)], check=True, capture_output=True, text=True)
            out[f"s{i}"] = np.array(r.stdout.split(), dtype=np.int32).reshape(ITERS, dof)
            out[f"case{i}"] = np.array([n, seed, dof], dtype=np.int32)
        out["count"] = np.int32(len(CASES))
        gxx = subprocess.run(["g++", "--version"], capture_output=True, text=True).stdout.splitlines()[0]
        out["compiler"] = np.array(gxx)
    np.savez_compressed(os.path.join(HERE, "lotbox3_golden.npz"), **out)
    print("wrote", len(CASES), "schedules,", gxx)


if __name__ == "__main__":
    sys.exit(main())
