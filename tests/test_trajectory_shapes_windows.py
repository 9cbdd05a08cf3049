"""The cases of test_gpu_batch_window_trajectory_shapes are what they are named for: window size, the factors that hold
samples and their sample counts, a noise of its own per factor, the warps and shared memory bw_trajectory_kernel gets,
the side of the smoother's 1e-10 pivot rule each near-singular factor is on, and the 50-digit judge agreeing with the
fp64 oracles where the GPU file uses it.  And the oracles' per-factor noise: one tuple reaches every factor as the same
object it did before, a list gives factor k its own, and the smoother's one-pass knot rotations are the bits of one
prefix integration per knot."""
import numpy as np
import pytest

from oracle import trajectory_oracle as to
import trajectory_mp_oracle as mpo
import trajectory_smoothing_oracle as tso
from test_gpu_batch_window_trajectory_shapes import (COV_MAX_N, MAX_FRAMES, MP_CASES, SPECS, smem_forward, sigma_T,
                                                     times, window)

# samples per factor, 0: none
EXPECT = {f"N{N}": (50,) * (N - 1) for N in range(1, 17)}
EXPECT.update({f"N{N}_{p}": tuple(50 if k in h else 0 for k in range(N - 1))
               for N in (7, 16) for p, h in (("none", ()), ("first", (0,)), ("last", (N - 2,)),
                                              ("all_but_first", range(1, N - 1)), ("all_but_last", range(N - 2)),
                                              ("alternate", range(0, N - 1, 2)), ("middle", ((N - 1) // 2,)))})
EXPECT.update({"N3_first": (50, 0), "mix": (1, 2, 3, 50, 250, 50, 2), "long": (400,) * 3, "sing": (2, 1, 50, 2),
               "gaps": (50, 50, 50, 48), "epoch": (50,) * 5, "offset": (50,) * 5})
# factor (case, k) -> smoother Sigma(T) positive definite
PD = {("sing", 0): True, ("sing", 1): False, ("sing", 3): True, ("long", 0): True, ("mix", 0): False, ("mix", 1): True}
RULE = 1e-10


def _frames(name):
    st = window(name)["st"]
    return np.concatenate([st.q, st.p, st.v, st.bg, st.ba], axis=1)


def test_every_case_is_the_window_it_is_named_for():
    assert set(EXPECT) == set(SPECS)
    for name, counts in EXPECT.items():
        c = window(name)
        assert c["N"] == SPECS[name]["N"] == len(counts) + 1, name
        got = tuple(0 if s is None else len(s) for s, _ in c["factors"])
        assert got == counts, (name, got)
        for s, t_end in c["factors"]:
            if s is not None:
                assert np.all(np.diff(s[:, 0]) > 0) and s[-1, 0] < t_end, name
    assert window("gaps")["factors"][1][0][0, 0] - window("gaps")["factors"][0][1] == pytest.approx(1e-9, rel=1e-3)
    assert window("gaps")["factors"][3][0][0, 0] - window("gaps")["factors"][2][1] == pytest.approx(1e-2)
    assert window("epoch")["factors"][0][0][0, 0] >= 1.7e9
    assert np.linalg.norm(window("offset")["st"].p[0]) > 4900.0
    fs = window("sing")["factors"]
    assert fs[0][1] - fs[0][0][-1, 0] == pytest.approx(1e-6, rel=1e-6)


def test_every_factor_has_its_own_noise():
    for name in SPECS:
        nz = [(k, n) for k, n in enumerate(window(name)["noises"]) if n is not None]
        for i in range(len(nz)):
            for j in range(i):
                assert any(not np.array_equal(a, b) for a, b in zip(nz[i][1], nz[j][1])), (name, i, j)
        for k, n in nz:
            for b in n:
                assert np.array_equal(b, b.T) and np.all(np.linalg.eigvalsh(b) > 0), name
                assert (np.count_nonzero(b - np.diag(np.diag(b))) > 0) == (k % 2 == 1), (name, k)   # odd k: full


def test_warps_and_shared_memory():
    warps = {name: max(1, s["N"] - 1) for name, s in SPECS.items()}
    assert min(warps.values()) == 1 and max(warps.values()) == MAX_FRAMES - 1
    assert smem_forward(1, False) == 4704 and smem_forward(1, True) == 11904
    assert smem_forward(8, True) == 95232 and smem_forward(15, True) == 178560
    assert smem_forward(15, True) <= 227 * 1024                          # the H100's opt-in shared memory per block
    assert [n for n in SPECS if SPECS[n]["N"] > COV_MAX_N] == ["N12", "N13", "N14", "N15", "N16"] + \
        [f"N16_{p}" for p in ("none", "first", "last", "all_but_first", "all_but_last", "alternate", "middle")]


def _pivot_ratio(S):
    """the smallest (R_jj^2 / S_jj) of chol_pd's factorisation, per diagonal block"""
    out = np.inf
    for a, b in ((0, 9), (9, 12), (12, 15)):
        B = S[a:b, a:b]
        n = len(B)
        R = np.zeros((n, n))
        for j in range(n - 1, -1, -1):
            d = B[j, j] - R[j, j + 1:] @ R[j, j + 1:]
            out = min(out, d / B[j, j])
            if d <= 0:
                return out
            R[j, j] = np.sqrt(d)
            for i in range(j):
                R[i, j] = (B[i, j] - R[i, j + 1:] @ R[j, j + 1:]) / R[j, j]
    return out


@pytest.mark.parametrize("case", sorted(PD))
def test_near_singular_factors_are_clear_of_the_pivot_rule(case):
    name, k = case
    S = sigma_T(window(name), _frames(name), k)
    r = _pivot_ratio(S)
    pd = tso.chol_pd(S[0:9, 0:9]) and tso.chol_pd(S[9:12, 9:12]) and tso.chol_pd(S[12:15, 12:15])
    print(f"{name} factor {k}: smallest pivot ratio {r:.2e} against {RULE:.0e}, positive definite {pd}")
    assert pd == PD[case]
    assert (r > 10 * RULE) if pd else (r < 0.1 * RULE)


@pytest.mark.parametrize("name", MP_CASES)
def test_fifty_digit_judge_agrees_with_the_oracle(name):
    c = window(name)
    F, frames = c["factors"], _frames(name)
    ts = times(name)
    fr = np.array([to.factor_of(t, F) for t in ts])
    i = np.flatnonzero(fr >= 0)[::7][:20]
    _, st, _ = to.trajectory(ts[i], frames, F, c["noises"])
    ref = np.array([mpo.state(frames[fr[r]], F[fr[r]][0], ts[r]) for r in i])
    e = (np.abs(st - ref) / (1.0 + np.abs(ref))).max()
    print(f"{name}: {len(i)} times, trajectory_oracle against 50 digits {e:.2e}")
    assert e < 1e-12


def _old_cross_cov(samples, t, t_end, bg, ba, noise):
    """tso.cross_cov as it was before _knot_rotations: one prefix integration per knot"""
    s = np.asarray(samples, dtype=np.float64).reshape(-1, 7)
    nz = np.concatenate([np.asarray(c, dtype=np.float64).reshape(9) for c in noise])
    d = to.delta(s, t, bg, ba, noise)
    P = np.block([[d["cov"], d["cov"]], [d["cov"], d["cov"]]])
    j = int(np.flatnonzero(s[:, 0] <= t)[-1])
    knots = list(s[:, 0]) + [float(t_end)]
    q, t0 = d["dq"], t
    for i in range(j, len(s)):
        P = tso._aug_step(P, q, s[i], knots[i + 1] - t0, bg, ba, nz)
        if i + 1 < len(s):
            q, t0 = to.delta(s, knots[i + 1], bg, ba, noise)["dq"], knots[i + 1]
    return P[0:15, 15:30]


def test_one_noise_reaches_every_factor_as_before():
    """With one noise tuple, noise_of hands every factor that very object, so trajectory() and smoothed() call delta()
    and gain() with exactly the argument they took before per-factor noise existed; with a list, factor k gets entry k
    and only factor k's rows move when it changes."""
    c = window("N5")
    F, frames = c["factors"], _frames("N5")
    noise = tuple(np.eye(3) * v for v in (1e-4, 2e-3, 3e-7, 4e-5))
    per = [noise, None, noise, noise]
    for k in range(4):
        assert to.noise_of(noise, k) is noise and to.noise_of(per, k) is per[k]
    other = (2.0 * noise[0], noise[1], noise[2], 3.0 * noise[3])     # not a uniform scale, which K would not see
    ts = times("N5")[::9]
    fr, st, _ = to.trajectory(ts, frames, F, noise)
    rng = np.random.default_rng(3)
    Sig = np.array([(lambda A: A @ A.T * 1e-4)(rng.normal(size=(15, 15))) for _ in range(5)])
    _, st1, cov1 = to.trajectory(ts, frames, F, noise, Sig)
    _, st2, cov2 = to.trajectory(ts, frames, F, [noise, noise, other, noise], Sig)
    J = rng.normal(size=(75, 75))
    joint = J @ J.T * 1e-4
    a = tso.smoothed(ts, frames, F, noise, joint)
    b = tso.smoothed(ts, frames, F, [noise, noise, other, noise], joint)
    assert np.array_equal(st, st1) and np.array_equal(st1, st2)        # the forward state does not read the noise
    for i, f in enumerate(fr):
        moved = f == 2 and ts[i] > F[2][0][0, 0]          # at its first sample the increment is empty
        assert moved != np.array_equal(cov1[i], cov2[i], equal_nan=True), (i, f)
        assert moved != np.array_equal(a[1][i], b[1][i]), (i, f)
    s, t_end = F[1]
    x = frames[1]
    for t in (s[0, 0], s[7, 0] + 1e-3, s[-1, 0], t_end):     # the one-pass knot rotations: the per-knot bits
        assert np.array_equal(tso.cross_cov(s, t, t_end, x[10:13], x[13:16], noise),
                              _old_cross_cov(s, t, t_end, x[10:13], x[13:16], noise)), t
