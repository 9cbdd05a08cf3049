"""Builds libpvio_b200.so in-tree with nvcc for sm_90a (H100; no JIT cache, no torch extension), so that the
package imports from the source tree.  Usage: python -m pvio_b200.build"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libpvio_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
         "-Xcompiler", "-fPIC", "-Xptxas", "-v", "--expt-relaxed-constexpr"]


def _extra(name):
    """per-file flags: OpenCV's float rounding and the reference's uncontracted fp64 on the device (no contraction);
    undistort.cu's host-side map builder without fused multiply-adds, which GCC forms by default where the target has
    them (aarch64)"""
    if name.endswith(("klt.cu", "detect.cu", "fmat.cu", "twoview.cu", "feature_track.cu",
                             "plane_ransac.cu", "imu_stream.cu")):
        return ["-fmad=false"]
    if name.endswith("undistort.cu"):
        return ["-Xcompiler", "-ffp-contract=off"]
    return []


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False, defines=(), out=None):
    """defines / out: the phase-stamp builds of tools/solve_stamps.py and tools/marg_stamps.py (-DPVIO_SOLVE_STAMPS,
    -DPVIO_MARG_STAMPS) -- objects go to a side directory, the product .so is untouched."""
    if defines or out:
        return _build_variant(list(defines), out)
    srcs = sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    hdrs.append(os.path.join(os.path.dirname(HERE), "include", "pvio_b200.h"))
    objs, jobs = [], []
    for s in srcs:
        src = os.path.join(CSRC, s)
        obj = os.path.join(CSRC, s[:-3] + ".o")
        objs.append(obj)
        if force or _stale(obj, [src] + hdrs):
            jobs.append((src, obj))

    def cc(job):
        src, obj = job
        extra = _extra(src)
        r = subprocess.run([NVCC] + FLAGS + extra + ["-c", src, "-o", obj], capture_output=True, text=True)
        return src, r

    with ThreadPoolExecutor(max_workers=4) as ex:
        for src, r in ex.map(cc, jobs):
            log = r.stdout + r.stderr
            with open(os.path.splitext(src)[0] + ".ptxas.log", "w") as f:
                f.write(log)
            if r.returncode != 0:
                sys.stderr.write(log)
                raise RuntimeError("nvcc failed on " + src)
            if verbose:
                print(log)
    if jobs or force or not os.path.exists(OUT):
        r = subprocess.run([NVCC, "-shared", "-o", OUT] + objs + ["-lcudart"], capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("link failed")
    return OUT


def _build_variant(defines, out):
    odir = os.path.join(HERE, "csrc", "_variants", os.path.basename(out))
    os.makedirs(odir, exist_ok=True)
    objs = []
    for s in sorted(f for f in os.listdir(CSRC) if f.endswith(".cu")):
        obj = os.path.join(odir, s[:-3] + ".o")
        extra = _extra(s)
        ref = os.path.join(CSRC, s[:-3] + ".o")
        names = [d.split("=")[0] for d in defines]
        text = open(os.path.join(CSRC, s)).read()
        uses = s == "api.cu" or any(n in text for n in names)      # api.cu includes every .cuh; other files: only if they name the define
        if not uses and os.path.exists(ref):
            objs.append(ref)
            continue
        r = subprocess.run([NVCC] + [f for f in FLAGS if f not in ("-Xptxas", "-v")] + extra + ["-D" + d for d in defines] +
                           ["-c", os.path.join(CSRC, s), "-o", obj], capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("nvcc failed on " + s)
        objs.append(obj)
    r = subprocess.run([NVCC, "-shared", "-o", out] + objs + ["-lcudart"], capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("link failed")
    return out


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
