"""ctypes loader for oracle/_build/libba_oracle.so (the C restatement of the reference's CPU path: the timed
baseline of bench.py and a second checker).  TEST / BASELINE INFRASTRUCTURE ONLY -- see oracle/ba_oracle.c.
The library takes the C-ABI's own window / state structures (include/pvio_b200.h), so the marshalling is the
one the product's host mirror uses (pvio_b200._lib.PackedArgs: plain ctypes mirrors of the header, no CUDA)."""
import ctypes as C
import os
import subprocess

import numpy as np

from pvio_b200 import _lib as L

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "libba_oracle.so")
_lib = None


def load(rebuild=False):
    global _lib
    if _lib is not None and not rebuild:
        return _lib
    src = os.path.join(_HERE, "ba_oracle.c")
    if rebuild or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
        subprocess.run(["make", "-s", "-C", _HERE] + (["-B"] if rebuild else []), check=True)
    lib = C.CDLL(_SO)
    WP, SP, OP, MP = C.POINTER(L.CWindow), C.POINTER(L.CState), C.POINTER(L.COptions), C.POINTER(L.CSummary)
    lib.ba_oracle_gn_step.argtypes = [WP, SP, C.c_double, L.c_f64p, L.c_f64p, L.c_f64p]
    lib.ba_oracle_solve.argtypes = [WP, SP, OP, MP]
    lib.ba_oracle_marginalize.argtypes = [WP, SP, C.c_int, L.c_f64p, L.c_f64p, L.c_f64p, L.c_f64p]
    lib.ba_oracle_batch.argtypes = [C.c_int, C.c_int, C.c_int, WP, SP, OP, C.c_double, C.c_int, L.c_f64p, L.c_f64p,
                                    C.POINTER(C.c_int64), L.c_f64p]
    lib.ba_oracle_usable_cores.restype = C.c_int
    _lib = lib
    return lib


def usable_cores():
    """CPUs this process may use: scheduler affinity capped by the cgroup quota (what the baseline's threads get)."""
    return int(load().ba_oracle_usable_cores())


def gn_step(win, st, mu=1e-8):
    lib = load()
    pa = L.PackedArgs(win, st)
    dx = np.zeros(15 * win.N + win.M)
    c0, c1 = C.c_double(), C.c_double()
    rc = lib.ba_oracle_gn_step(C.byref(pa.cw), C.byref(pa.cs), mu, L.ptr(dx), C.byref(c0), C.byref(c1))
    assert rc == 0
    return dict(dx=dx, cost=c0.value, new_cost=c1.value)


def solve(win, st, max_iter=10, radius0=0.0, alias_bias=True):
    """Returns (frames [N,16], rho [M], summary dict)."""
    lib = load()
    pa = L.PackedArgs(win, st)
    opt = L.COptions(max_iter, 0.0, 1 if alias_bias else 0, 0, radius0)
    sm = L.CSummary()
    lib.ba_oracle_solve(C.byref(pa.cw), C.byref(pa.cs), C.byref(opt), C.byref(sm))
    return pa.keep["frames"].copy(), pa.keep["rho"].copy(), {k: getattr(sm, k) for k, _ in L.CSummary._fields_}


def marginalize(win, st, index=0):
    lib = load()
    pa = L.PackedArgs(win, st)
    d = 15 * (win.N - 1)
    S, e, H, b = np.zeros((d, d)), np.zeros(d), np.zeros((d, d)), np.zeros(d)
    rc = lib.ba_oracle_marginalize(C.byref(pa.cw), C.byref(pa.cs), index, L.ptr(S), L.ptr(e), L.ptr(H), L.ptr(b))
    assert rc == 0
    return S, e, H, b


def batch(kind, win, st, n_windows, n_threads=0, mu=1e-8, max_iter=10, index=0, want=False):
    """n_windows independent copies of one problem over POSIX threads.  kind: "gn_step" | "solve" | "marginalize".
    Returns (threads_used, total iterations [solve] or n_windows, optional outputs)."""
    lib = load()
    pa = L.PackedArgs(win, st)
    k = {"gn_step": 0, "solve": 1, "marginalize": 2}[kind]
    opt = L.COptions(max_iter, 0.0, 1, 0, 0.0)
    dx = np.zeros((n_windows, 15 * win.N + win.M)) if k == 0 else None
    costs = np.zeros((n_windows, 2)) if k == 0 else None
    iters = np.zeros(n_windows, dtype=np.int64) if k == 1 else None
    fcost = np.zeros(n_windows) if k == 1 else None
    used = lib.ba_oracle_batch(k, n_windows, n_threads, C.byref(pa.cw), C.byref(pa.cs), C.byref(opt), mu, index,
                               L.ptr(dx), L.ptr(costs), L.ptr(iters), L.ptr(fcost))
    units = int(iters.sum()) if k == 1 else n_windows
    return (used, units, dict(dx=dx, costs=costs, iters=iters, final_costs=fcost)) if want else (used, units)


def gn_step_batch(win, st, n_windows, n_threads=0, mu=1e-8):
    """n_windows independent copies over POSIX threads; returns (dx, costs, threads_used)."""
    used, _, out = batch("gn_step", win, st, n_windows, n_threads, mu=mu, want=True)
    return out["dx"], out["costs"], used
