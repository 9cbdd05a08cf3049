"""Writes tests/golden/lotbox_golden.npz: the sample schedules of PVIO's Ransac::solve (utility/ransac.h), drawn by a
small C++ program compiled here with g++ against <random> only -- a LotBox of n lots over std::default_random_engine
and std::uniform_int_distribution<size_t>, refilled every iteration.  Run: python tests/golden/make_lotbox_golden.py"""
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = [(n, seed, dof) for n in (4, 5, 6, 50, 300, 2000) for seed in (648, 0) for dof in (4, 5)]
ITERS = 1000

SRC = r"""
#include <cstdio>
#include <cstdlib>
#include <random>
#include <utility>
#include <vector>
int main(int argc, char **argv) {
    const size_t n = std::strtoul(argv[1], nullptr, 10), dof = std::strtoul(argv[3], nullptr, 10),
                 iters = std::strtoul(argv[4], nullptr, 10);
    const unsigned seed = (unsigned)std::strtol(argv[2], nullptr, 10);
    std::vector<size_t> lots(n);
    for (size_t i = 0; i < n; ++i) lots[i] = i;
    std::default_random_engine engine;
    engine.seed(seed);
    std::uniform_int_distribution<size_t> dist;
    for (size_t it = 0; it < iters; ++it) {
        size_t cap = 0;
        for (size_t s = 0; s < dof; ++s) {
            size_t v;
            if (n - cap > 1) {
                const size_t j = dist(engine, std::uniform_int_distribution<size_t>::param_type(cap, n - 1));
                std::swap(lots[cap], lots[j]);
                v = lots[cap];
            } else {
                v = lots[n - 1];
            }
            ++cap;
            std::printf("%zu\n", v);
        }
    }
    return 0;
}
"""


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
    np.savez_compressed(os.path.join(HERE, "lotbox_golden.npz"), **out)
    print("wrote", len(CASES), "schedules,", gxx)


if __name__ == "__main__":
    sys.exit(main())
