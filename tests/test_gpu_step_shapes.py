"""The batched Gauss-Newton step and the trust-region solve on both sides of every launch-shape choice api.cu makes per
call, at the window shapes and handle capacities at the kernels' granules.

The choices and what pins each side here:
  * sweep_grid_x (n * 2 < SMs: 16 CTAs per window with fp64 atomics, 7 launches per step; otherwise one CTA per window,
    5 launches) and gn_step_parts (from 7 windows per SM: sub-batches on two streams, 5 launches each) are observable
    through kernel_launches, which every batched step here asserts.  The band edges come from the device's SM count.
  * run_solve's lean (solve_kernel_visual) and wide (solve_kernel) kernels and lin_part_fits' shared-memory sums and jr
    records path are not observable through the ABI.  Their cases sit well clear of the thresholds: 14 free frames
    (D = 84, the lean kernel) against 15 and 16 (D = 90 and 96, the wide one); 500 landmarks (shared sums) against 1,200
    and 3,000 (records), as test_gpu_step_records establishes.
  * The latency path of the solve loop (n * 2 < SMs: one captured graph) sizes its launches by the handle's capacity.

Bars (DESIGN §2): dx within 1e-5 relative of the oracle step (2e-5 for 16-frame fp32 windows), cost within 2e-6, the
coordinates of fixed frames exactly 0; replicas bit-identical on the fp32 batched path, within 1e-10 on the fp64 one and
within 1e-9 on the latency path (fp64 atomics from 16 CTAs); solves with the bars of test_solve_matches_oracle_loop.
Windows whose gauge is not fixed by two constant frames (one or no fixed frame of a visual window) are stepped with
mu = 1e-2, so that the damped system is conditioned well enough for fp32 Jacobians; the oracle takes the same mu."""
import ctypes as C
import functools
import math

import numpy as np
import pytest

from oracle import ba_oracle as bo
from synthetic import synth
from pvio_b200 import _lib as L
from pvio_b200.bundle_adjustor import BundleAdjustor, PvioB200Error

pytestmark = pytest.mark.gpu

MU = 1e-8
MU_GAUGE = 1e-2
CHUNK, MAX_CHUNKS = 32, 96            # ba_lin.cuh kChunk, ba_types.h kMaxChunks: a window holds <= 3,072 landmarks


# ------------------------------------------------------------------ window builders (pinned by test_step_shapes_windows)
def shape_window(N, M, fixed=None, seed=1000, staggered=False):
    """A cfg2 window of N frames and M landmarks; fixed: the constant frames (default: cfg2's frames 0 and 1)"""
    w, st, _ = synth.make_cfg2(N=N, M=M, seed=seed, staggered=staggered)
    if fixed is not None:
        w.frame_fixed[:] = 0
        w.frame_fixed[list(fixed)] = 1
    return w, st


def n_free(w):
    return int(w.N - np.count_nonzero(w.frame_fixed))


def chunk_count(w):
    """api.cu pack_window's chunks: runs of <= 32 landmarks of one anchor, landmarks sorted by anchor"""
    a = np.sort(np.asarray(w.lm_anchor, dtype=np.int64), kind="stable")
    return int(sum(math.ceil(np.count_nonzero(a == x) / CHUNK) for x in np.unique(a)))


def segment_rows(w):
    """rows of 32 of the frame-major table (ba_fobs.cuh): per (target, anchor) segment, its blocks rounded up to 32"""
    cnt = {}
    for l in range(w.M):
        for k in range(int(w.lm_obs_begin[l]), int(w.lm_obs_begin[l + 1])):
            key = (int(w.obs_frame[k]), int(w.lm_anchor[l]))
            cnt[key] = cnt.get(key, 0) + 1
    return sum((c + 31) // 32 for c in cnt.values())


def step_mu(w):
    """visual windows with fewer than two constant frames leave the scale (and the gauge) to the damping, and so do
    windows with fewer residual rows than free coordinates"""
    if w.use_inertial or n_free(w) == 0:
        return MU
    return MU_GAUGE if np.count_nonzero(w.frame_fixed) < 2 or 2 * w.K < 6 * n_free(w) + w.M else MU


# name -> builder; every window a test steps is one of these, so that the oracle runs once per window
SHAPE_M = (0, 1, 3, 4, 5, 31, 32, 33, 63, 64, 65, 127, 128, 129, 3072)
SHAPE_FREE = {0: tuple(range(16)), 1: tuple(f for f in range(16) if f != 9), 14: (3, 11), 15: (7,), 16: ()}
CASES = {f"M{m}": functools.partial(shape_window, 4, m, seed=1100 + m) for m in SHAPE_M}
CASES.update({
    "N2": functools.partial(shape_window, 2, 64, fixed=(0,), seed=1201),
    "N3": functools.partial(shape_window, 3, 64, seed=1202),
    "N16": functools.partial(shape_window, 16, 240, seed=12, staggered=True),
})
CASES.update({f"free{k}": functools.partial(shape_window, 16, 96, fixed=fx, seed=1300 + k, staggered=True)
              for k, fx in SHAPE_FREE.items()})
CASES.update({
    "M3073": functools.partial(shape_window, 4, 3073, seed=1400),               # a 97th chunk: rejected
    "cfg2": lambda: synth.make_cfg2()[:2],
    "het0": lambda: synth.make_cfg2(N=10, M=500, seed=41)[:2],
    "het1": lambda: synth.make_cfg2(N=10, M=420, staggered=True, seed=42)[:2],
    "het2": functools.partial(shape_window, 8, 300, fixed=(0, 5), seed=43),
    "het3": lambda: synth.make_cfg2(N=9, M=350, staggered=True, seed=44)[:2],
    "small0": lambda: synth.make_cfg2(N=6, M=80, seed=51)[:2],
    "small1": lambda: synth.make_cfg2(N=5, M=40, staggered=True, seed=52)[:2],
    "small2": functools.partial(shape_window, 8, 100, fixed=(0, 5), seed=53),
    "lm3000": lambda: synth.make_cfg2(N=4, M=3000, seed=77)[:2],
    "free15_16": functools.partial(shape_window, 16, 240, fixed=(7,), seed=12, staggered=True),
    "inertial": lambda: synth.make_cfg3(N=6, M=100, seed=44)[:2],
    "plane": lambda: synth.make_cfg4(N=6, M=60, seed=24, tracks_per_plane=20)[:2],
})
CASES.update({f"cap{m}": functools.partial(shape_window, 4, m, seed=1500 + m) for m in (65, 66, 67)})
HET = ("het0", "het1", "het2", "het3")
SMALL = ("small0", "small1", "small2")


@functools.lru_cache(maxsize=None)
def window(name):
    return CASES[name]()


@functools.lru_cache(maxsize=None)
def oracle(name, mu):
    w, st = window(name)
    return bo.gn_step(w, st, mu=mu, schur=True)


def case(name):
    """(window, state, oracle step at the window's mu, mu)"""
    w, st = window(name)
    mu = step_mu(w)
    return w, st, oracle(name, mu), mu


# ------------------------------------------------------------------ device helpers
@pytest.fixture(scope="module")
def sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def half(sm):
    return (sm + 1) // 2            # the smallest batch of the batched path: n * 2 >= SMs


def _rel(a, b):
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)


WORST = {}


def _note(band, dx_err, cost_err):
    d, c = WORST.get(band, (0.0, 0.0))
    WORST[band] = (max(d, dx_err), max(c, cost_err))


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for band, (d, c) in sorted(WORST.items()):
        print(f"step shapes: {band}: worst dx rel err {d:.2e}, worst cost rel err {c:.2e}")


def _set(b, names, n):
    """slot i <- window names[i % len(names)] for i < n"""
    packs = {nm: L.PackedArgs(*case(nm)[:2]) for nm in set(names)}
    for i in range(n):
        p = packs[names[i % len(names)]]
        rc = b.lib.pvio_b200_batch_set_window(b.h, i, C.byref(p.cw), C.byref(p.cs))
        assert rc == 0, b.lib.pvio_b200_last_error(b.h).decode()
    b.batch_upload(n)


def _step(b, n, mu, stride):
    l0 = b.kernel_launches
    b.batch_gn_step(n, mu, apply=False)
    launches = b.kernel_launches - l0
    dx, costs = b.batch_download(n, stride)
    return dx, costs, launches


def _launches(sm, n, parts=1):
    return 7 if n * 2 < sm else 5 * parts


def _check(band, name, dx_row, cost, mu=None):
    w, st, ref, mu0 = case(name)
    if mu is not None and mu != mu0:
        ref = oracle(name, mu)
    n = 15 * w.N + w.M
    d = dx_row[:n]
    # 16-frame windows and windows with fewer residual rows than free coordinates (M = 1): the fp32 Jacobians' 2e-5
    tol = 2e-5 if w.N == 16 or 2 * w.K < 6 * n_free(w) + w.M else 1e-5
    e, ec = _rel(d, ref["dx"]), abs(cost - ref["cost"]) / max(ref["cost"], 1e-300)
    _note(band, e, ec)
    assert e < tol, (band, name, e)
    assert abs(cost - ref["cost"]) <= 2e-6 * ref["cost"], (band, name, cost, ref["cost"])
    assert np.all(d[~ref["free"]] == 0.0), (band, name)


def _replicas(dx, costs, rows, pipeline_fp64, latency):
    """rows of one window: bit-identical (fp32 batched), 1e-10 (fp64 batched) or 1e-9 (latency path) apart"""
    r0 = rows[0]
    for r in rows[1:]:
        if latency:
            assert _rel(dx[r], dx[r0]) < 1e-9, (r, r0)
        elif pipeline_fp64:
            assert np.allclose(dx[r], dx[r0], rtol=1e-10, atol=0), (r, r0)
        else:
            assert np.array_equal(dx[r], dx[r0]) and np.array_equal(costs[r], costs[r0]), (r, r0)


def _fp64(b):
    """turn the handle's records to fp64: pack an inertial window once (into its last slot)"""
    w, st = case("inertial")[:2]
    b.batch_set(b.max_windows - 1, w, st)


# ------------------------------------------------------------------ 1. batch-size bands
def _band_sizes(sm):
    h = half(sm)
    return {"n=1": 1, "n=63": 63, "n=64": 64, "n=65": 65, "half-1": h - 1, "half": h, "7sm-1": 7 * sm - 1, "7sm": 7 * sm}


BANDS = ("n=1", "n=63", "n=64", "n=65", "half-1", "half", "7sm-1", "7sm")


@pytest.fixture(scope="module")
def band_ba(sm):
    b = BundleAdjustor(max_windows=7 * sm, max_frames=10, max_landmarks=512, max_obs=4608)
    yield b
    b.close()


@pytest.fixture(scope="module")
def batched_bits(band_ba, sm):
    """the batched path's dx and costs per window kind (at n = ceil(SMs / 2)): a window's bits do not depend on n or
    on its position in the batch"""
    n = max(half(sm), 64)
    out = {}
    for names in (("cfg2",), HET):
        _set(band_ba, names, n)
        dx, costs, _ = _step(band_ba, n, MU, 15 * 10 + 512)
        for k, nm in enumerate(names):
            out[nm] = (dx[k].copy(), costs[k].copy())
    return out


@pytest.mark.parametrize("band", BANDS)
def test_step_at_batch_size_band(band_ba, sm, batched_bits, band):
    n = _band_sizes(sm)[band]
    if band in ("n=64", "n=65") and not n * 2 < sm:
        pytest.skip(f"64 <= n < SMs / 2 is empty on a {sm}-SM device")
    if n < 1 or n > band_ba.max_windows:
        pytest.skip(f"no batch of {n} windows on a {sm}-SM device")
    latency = n * 2 < sm
    parts = 2 if n >= 7 * sm else 1
    label = "latency" if latency else ("split" if parts > 1 else "batched")
    stride = 15 * 10 + 512
    for names in (("cfg2",), HET):
        _set(band_ba, names, n)
        dx, costs, launches = _step(band_ba, n, MU, stride)
        assert launches == _launches(sm, n, parts), (band, launches)
        for k, nm in enumerate(names):
            rows = list(range(k, n, len(names)))
            if not rows:
                continue
            for r in (rows[0], rows[-1]):
                _check(f"band {band} ({label})", nm, dx[r], costs[r, 0])
            _replicas(dx, costs, rows, False, latency)
            if not latency:
                ref_dx, ref_c = batched_bits[nm]
                assert np.array_equal(dx[rows[-1]], ref_dx) and np.array_equal(costs[rows[-1]], ref_c), (band, nm)


def test_forced_split_is_clamped(band_ba, sm):
    """4 sub-batches forced on 3 * max(SMs, 64) windows: gn_step_parts clamps them to 3 (every part keeps at least
    max(SMs, 64) windows), and the windows keep their batched bits"""
    n = 3 * max(sm, 64)
    if n > band_ba.max_windows:
        pytest.skip(f"{n} windows exceed the band handle on a {sm}-SM device")
    _set(band_ba, HET, n)
    assert band_ba.lib.pvio_b200_internal_set_step_split(band_ba.h, 4) == 0
    try:
        dx, costs, launches = _step(band_ba, n, MU, 15 * 10 + 512)
    finally:
        assert band_ba.lib.pvio_b200_internal_set_step_split(band_ba.h, 0) == 0
    assert launches == 15
    for k, nm in enumerate(HET):
        rows = list(range(k, n, len(HET)))
        _check("forced split (3 parts)", nm, dx[rows[-1]], costs[rows[-1], 0])
        _replicas(dx, costs, rows, False, False)


@pytest.mark.parametrize("which", ("n=1", "n=64", "n=65", "half"))
def test_batch_solve_band_matches_single_window_solve(sm, which):
    """batch_solve of three kinds (one starts converged) against each window's own single-window solve: the same
    kernels and decisions on the latency path (bars of test_batch_solve_matches_single_window_solve), the oracle-loop
    bars where the batch runs one CTA per window and the lean solve"""
    n = {"n=1": 1, "n=64": 64, "n=65": 65, "half": half(sm)}[which]
    if which in ("n=64", "n=65") and not n * 2 < sm:
        pytest.skip(f"64 <= n < SMs / 2 is empty on a {sm}-SM device")
    b = BundleAdjustor(max_windows=max(n, 3), max_frames=8, max_landmarks=160, max_obs=1200)
    try:
        kinds = [case(nm)[:2] for nm in SMALL]
        conv, _ = b.solve(*kinds[1], max_iterations=40)
        kinds[1] = (kinds[1][0], conv)
        singles = [b.solve(w, st, max_iterations=7) for w, st in kinds]
        for i in range(n):
            b.batch_set(i, *kinds[i % 3])
        b.batch_upload(n)
        b.batch_solve(n, max_iterations=7)
        frames, rho, sm_out = b.batch_download_state(n, 8, 160)
    finally:
        b.close()
    latency = n * 2 < sm
    for i in sorted({0, 1, 2, n - 3, n - 2, n - 1} & set(range(n))):
        w, st = kinds[i % 3]
        ref_state, ref_sum = singles[i % 3]
        assert sm_out[i]["iterations"] == ref_sum["iterations"] and sm_out[i]["termination"] == ref_sum["termination"], i
        if latency:
            assert abs(sm_out[i]["final_cost"] - ref_sum["final_cost"]) <= 1e-9 * ref_sum["final_cost"], i
            assert np.allclose(frames[i, :w.N, 4:7], ref_state.p, rtol=0, atol=1e-9), i
            assert np.allclose(rho[i, :w.M], ref_state.rho, rtol=1e-9, atol=0), i
        else:
            assert abs(sm_out[i]["final_cost"] - ref_sum["final_cost"]) <= 1e-5 * ref_sum["final_cost"], i
            move = np.linalg.norm(ref_state.p - st.p)
            assert np.linalg.norm(frames[i, :w.N, 4:7] - ref_state.p) < 1e-5 * max(move, 1e-3) + 1e-9, i
            assert np.linalg.norm(rho[i, :w.M] - ref_state.rho) < 1e-5 * np.linalg.norm(ref_state.rho - st.rho) + 1e-9, i


# ------------------------------------------------------------------ 2. one window decides for the batch
DECIDERS = {"fp32": ("lm3000", "free15_16"), "fp64": ("lm3000", "free15_16", "inertial", "plane")}


@pytest.mark.parametrize("precision,decider", [(p, d) for p, ds in DECIDERS.items() for d in ds])
def test_deciding_window_in_a_visual_batch(sm, precision, decider):
    """One window that moves the whole batch to other kernels -- 3,000 landmarks (the jr records path), 15 free frames
    of 16 (the wide solve), an inertial or a plane window (the wide solve; the fp64 records on an fp32 handle) -- in
    the middle of a batch of small visual windows.  Every window against its own oracle step."""
    n = half(sm)
    mcap = 3000 if decider == "lm3000" else 240
    b = BundleAdjustor(max_windows=n + 1, max_frames=16, max_landmarks=mcap, max_obs=9000)
    try:
        if precision == "fp64":
            _fp64(b)
        names = [SMALL[i % 3] for i in range(n)]
        names[n // 2] = decider
        _set(b, names, n)
        dx, costs, launches = _step(b, n, MU_GAUGE, 15 * 16 + mcap)
        fp64 = precision == "fp64" or decider in ("inertial", "plane")
    finally:
        b.close()
    assert launches == _launches(sm, n)
    band = f"decider {decider} ({precision} handle)"
    for i in sorted({0, 1, 2, n // 2, n - 3, n - 2, n - 1}):     # every kind, first and last; the decider
        _check(band, names[i], dx[i], costs[i, 0], mu=MU_GAUGE)
    for k in range(3):
        rows = [i for i in range(n) if names[i] == SMALL[k]]
        _replicas(dx, costs, rows, fp64, False)


# ------------------------------------------------------------------ 3. window shapes
SHAPES = [f"M{m}" for m in SHAPE_M] + ["N2", "N3", "N16"] + [f"free{k}" for k in SHAPE_FREE]


@pytest.fixture(scope="module", params=("fp32", "fp64"))
def shape_ba(request, sm):
    b = BundleAdjustor(max_windows=half(sm) + 1, max_frames=16, max_landmarks=3076, max_obs=9300)
    if request.param == "fp64":
        _fp64(b)
    b.precision = request.param
    yield b
    b.close()


@pytest.mark.parametrize("name", SHAPES)
def test_window_shape_alone_and_replicated(shape_ba, sm, name):
    """Each shape alone (the latency path) and as a batch of ceil(SMs / 2) replicas (one CTA per window)"""
    w, st, ref, mu = case(name)
    fp64 = shape_ba.precision == "fp64"
    stride = 15 * w.N + w.M
    for n in (1, half(sm)):
        _set(shape_ba, (name,), n)
        dx, costs, launches = _step(shape_ba, n, mu, stride)
        assert launches == _launches(sm, n)
        latency = n * 2 < sm
        band = f"shape {'alone' if n == 1 else 'replicated'} ({shape_ba.precision})"
        for r in (0, n - 1):
            _check(band, name, dx[r], costs[r, 0])
        _replicas(dx, costs, list(range(n)), fp64, latency)
        if n_free(w) == 0:
            assert np.all(dx[:, :15 * w.N] == 0.0)
        if w.M == 0:                       # no residual: no step, no cost
            assert np.all(dx == 0.0) and np.all(costs[:, 0] == 0.0)
            assert ref["cost"] == 0.0 and np.all(ref["dx"] == 0.0)


def test_97th_chunk_is_rejected_and_changes_nothing(shape_ba, sm):
    """3,073 landmarks of one anchor need a 97th chunk: batch_set and gn_step refuse them; the uploaded windows step
    to the same results afterwards, and their download is shaped by the windows that were accepted"""
    w3, s3 = case("M3073")[:2]
    assert chunk_count(w3) == MAX_CHUNKS + 1
    n = half(sm)
    _set(shape_ba, ("M3072",), n)
    w, st, _, mu = case("M3072")
    dx0, c0, _ = _step(shape_ba, n, mu, 15 * w.N + w.M)
    pa = L.PackedArgs(w3, s3)
    assert shape_ba.lib.pvio_b200_batch_set_window(shape_ba.h, 0, C.byref(pa.cw), C.byref(pa.cs)) == L.EINVAL
    assert "chunks" in shape_ba.lib.pvio_b200_last_error(shape_ba.h).decode()
    with pytest.raises(PvioB200Error, match=f"error {L.EINVAL}"):
        shape_ba.gn_step(w3, s3)
    # the download after the rejection writes exactly the uploaded windows' rows: a sentinel behind the last row stays
    stride = 15 * w.N + w.M
    shape_ba.batch_gn_step(n, mu, apply=False)
    buf, c1 = np.full(n * stride + 8, np.nan), np.zeros((n, 2))
    assert shape_ba.lib.pvio_b200_batch_download(shape_ba.h, n, L.ptr(buf), stride, L.ptr(c1)) == 0
    assert np.all(np.isnan(buf[n * stride:]))
    dx1 = buf[:n * stride].reshape(n, stride)
    if shape_ba.precision == "fp32":
        assert np.array_equal(dx0, dx1) and np.array_equal(c0, c1)
    else:                                  # the fp64 pipeline's cross-warp sums round in the order they arrive
        assert np.allclose(dx1, dx0, rtol=1e-10, atol=0) and np.allclose(c1, c0, rtol=1e-10, atol=0)


# ------------------------------------------------------------------ 4. capacities
@pytest.mark.parametrize("name", ("cap65", "cap66", "cap67"))
def test_tight_capacities(sm, name):
    """max_landmarks = M with M = 1, 2, 3 (mod 4) (the Schur copies read the rounded-up padding), max_obs = K and an
    odd max_windows whose last slot is in use, alone and batched"""
    w, st, _, mu = case(name)
    W = half(sm) | 1
    b = BundleAdjustor(max_windows=W, max_frames=w.N, max_landmarks=w.M, max_obs=w.K)
    try:
        for n in (1, W):
            _set(b, (name,), n)
            dx, costs, launches = _step(b, n, mu, 15 * w.N + w.M)
            assert launches == _launches(sm, n)
            for r in (0, n - 1):
                _check(f"capacity M = max_landmarks (n = {'1' if n == 1 else 'W'})", name, dx[r], costs[r, 0])
            _replicas(dx, costs, list(range(n)), False, n * 2 < sm)
    finally:
        b.close()


def test_sixteen_frame_capacity_with_small_windows(sm):
    """max_frames = 16 with 4-frame windows: the strides of the handle, the shapes of the windows"""
    names = ("M64", "M129", "N3")
    n = half(sm)
    b = BundleAdjustor(max_windows=n, max_frames=16, max_landmarks=160, max_obs=600)
    try:
        for m in (1, n):
            _set(b, names, m)
            dx, costs, launches = _step(b, m, MU, 15 * 16 + 160)
            assert launches == _launches(sm, m)
            for k, nm in enumerate(names[:m]):
                _check("max_frames 16, N <= 4", nm, dx[k], costs[k, 0])
    finally:
        b.close()


BIG_CAPS = (8000, 65534)


@pytest.fixture(scope="module")
def right_sized(sm):
    """the reference results of a handle sized to the windows (max_landmarks 160)"""
    b = BundleAdjustor(max_windows=max(half(sm), 8), max_frames=8, max_landmarks=160, max_obs=1200)
    out = {}
    try:
        kinds = [case(nm)[:2] for nm in SMALL]
        out["solve"] = [b.solve(w, st, max_iterations=6) for w, st in kinds]
        n = half(sm)
        _set(b, SMALL, n)
        out["step"] = _step(b, n, MU, 15 * 8 + 160)
    finally:
        b.close()
    return out


def _solve_close(out, summ, ref_state, ref_sum, st):
    assert summ["iterations"] == ref_sum["iterations"]
    assert abs(summ["final_cost"] - ref_sum["final_cost"]) <= 1e-5 * ref_sum["final_cost"]
    move = np.linalg.norm(ref_state.p - st.p)
    assert np.linalg.norm(out[0] - ref_state.p) < 1e-5 * max(move, 1e-3) + 1e-9
    assert np.linalg.norm(out[1] - ref_state.rho) < 1e-5 * np.linalg.norm(ref_state.rho - st.rho) + 1e-9


@pytest.mark.parametrize("mcap", BIG_CAPS)
def test_large_max_landmarks(sm, right_sized, mcap):
    """Handles far above the 3,072 landmarks a window can hold.  The latency path (solve, batch_solve of few windows,
    a resident solve, a step of few windows) sizes its launches by the capacity, so it must stay within the device's
    shared memory; the batched step's shapes follow the windows, so its results equal the right-sized handle's bits."""
    from pvio_b200.batch_window import BatchWindows
    from test_gpu_batch_window import _feed_window
    n = half(sm)
    kinds = [case(nm)[:2] for nm in SMALL]
    b = BundleAdjustor(max_windows=max(n, 8), max_frames=8, max_landmarks=mcap, max_obs=1200)
    try:
        for (w, st), (ref_state, ref_sum) in zip(kinds, right_sized["solve"]):
            out, summ = b.solve(w, st, max_iterations=6)
            _solve_close((out.p, out.rho), summ, ref_state, ref_sum, st)
        for m in (1, 8):
            for i in range(m):
                b.batch_set(i, *kinds[i % 3])
            b.batch_upload(m)
            b.batch_solve(m, max_iterations=6)
            frames, rho, sms = b.batch_download_state(m, 8, 160)
            for i in range(m):
                w, st = kinds[i % 3]
                ref_state, ref_sum = right_sized["solve"][i % 3]
                _solve_close((frames[i, :w.N, 4:7], rho[i, :w.M]), sms[i], ref_state, ref_sum, st)
        _set(b, SMALL, 1)
        dx, costs, launches = _step(b, 1, MU, 15 * 8 + 160)
        assert launches == _launches(sm, 1)
        _check(f"max_landmarks {mcap} (n = 1)", SMALL[0], dx[0], costs[0, 0])
        _set(b, SMALL, n)
        dx, costs, launches = _step(b, n, MU, 15 * 8 + 160)
        assert launches == _launches(sm, n)
        ref_dx, ref_c, _ = right_sized["step"]
        assert np.array_equal(dx, ref_dx) and np.array_equal(costs, ref_c)
    finally:
        b.close()
    # a resident solve of two slots on such a handle against the same on a right-sized one
    res = []
    for cap in (mcap, 160):
        r = BundleAdjustor(max_windows=2, max_frames=8, max_landmarks=cap, max_obs=1200)
        try:
            bw = BatchWindows(r)
            for s in range(2):
                _feed_window(bw, s, *kinds[s])
            summ = bw.solve([0, 1], max_iterations=6)
            res.append((summ, bw.download(range(2), 160)))
        finally:
            r.close()
    (sb, db), (ss, ds) = res
    for s in range(2):
        assert sb[s]["iterations"] == ss[s]["iterations"] and sb[s]["iterations"] > 0
        assert abs(sb[s]["final_cost"] - ss[s]["final_cost"]) <= 1e-5 * ss[s]["final_cost"]
        move = np.linalg.norm(ds[s]["frames"][:, 4:7] - kinds[s][1].p)
        assert np.linalg.norm(db[s]["frames"][:, 4:7] - ds[s]["frames"][:, 4:7]) < 1e-5 * max(move, 1e-3) + 1e-9
