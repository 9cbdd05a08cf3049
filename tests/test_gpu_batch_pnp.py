"""pvio_b200_batch_pnp_solve: visual_inertial_pnp (pvio/src/pvio/estimation/pnp.cpp:32-100) for a whole batch of
independent problems in one kernel launch, one CTA per problem.  Checked against the fp64 oracle, against the single
call beyond one wave of the GPU, for its launch count, its rejections and the growth of its staging buffers."""
import ctypes as C

import numpy as np
import pytest

from oracle import pnp_oracle as po
from synthetic import synth
from pvio_b200 import _lib, pnp
from pvio_b200.bundle_adjustor import BundleAdjustor
from pvio_b200._lib import EINVAL

pytestmark = pytest.mark.gpu

COST_TOL, STATE_TOL = 1e-9, 1e-8      # the bars of test_gpu_pnp.py


@pytest.fixture(scope="module")
def ba():
    b = BundleAdjustor(max_windows=1, max_frames=4, max_landmarks=16, max_obs=64)
    yield b
    b.close()


def _problem(cal, inertial, npts, seed):
    """A make_pnp problem with npts points (0: the IMU prior alone)."""
    d = synth.make_pnp(seed=seed, n_points=max(npts, 1), cal=cal, use_inertial=inertial)
    d['pts'], d['zs'] = d['pts'][:npts], d['zs'][:npts]
    return d


# EUROC and TUMVI, inertial and visual-only, 0 (inertial only) to 400 points
MIX = [(synth.EUROC, True, 0), (synth.TUMVI, True, 0), (synth.EUROC, True, 8), (synth.TUMVI, False, 8),
       (synth.EUROC, False, 40), (synth.TUMVI, True, 40), (synth.EUROC, True, 150), (synth.TUMVI, True, 150),
       (synth.EUROC, False, 150), (synth.TUMVI, False, 400), (synth.EUROC, True, 400), (synth.TUMVI, True, 8)]


def _mix():
    return [_problem(cal, inertial, npts, 700 + 13 * i) for i, (cal, inertial, npts) in enumerate(MIX)]


def _oracle(d, r0):
    kw = dict(radius0=r0) if r0 > 0 else {}
    return po.pnp_solve(d['frame'], d['last'], d['imu'], d['pts'].reshape(-1, 3), d['zs'].reshape(-1, 2), d['cam_q'],
                        d['cam_p'], d['imu_q'], d['imu_p'], d['W'], d['use_inertial'], **kw)


def _single(ba, d, r0=0.0):
    return pnp.visual_inertial_pnp(ba, d['frame'], d['last'], d['imu'], d['pts'], d['zs'], d['cam_q'], d['cam_p'],
                                   d['imu_q'], d['imu_p'], d['W'], d['use_inertial'], initial_radius=r0)


def _check_oracle(d, xg, sg, r0):
    xr, sr = _oracle(d, r0)
    assert sg['iterations'] == sr['iterations'] and sg['accepted_steps'] == sum(sr['accepted'])
    assert abs(sg['initial_cost'] - sr['initial_cost']) <= COST_TOL * sr['initial_cost']
    if len(d['pts']) == 0:
        # the IMU prior alone is met exactly: its final cost (~1e-23) is rounding noise, so the state is held to the
        # absolute bar of test_gpu_pnp.py's inertial-only case instead
        assert np.linalg.norm(xg - xr) < STATE_TOL
        return
    assert abs(sg['final_cost'] - sr['final_cost']) <= COST_TOL * sr['final_cost']
    move = np.linalg.norm(xr - d['frame'])
    assert np.linalg.norm(xg - xr) < STATE_TOL * max(move, 1e-3)
    if not d['use_inertial']:
        assert np.array_equal(xg[7:], d['frame'][7:])          # v, bg, ba are not parameters (pnp.cpp:46-54)


@pytest.mark.parametrize("r0", [0.0, 3.0])
def test_batch_matches_oracle(ba, r0):
    probs = _mix()
    xs, sums = pnp.batch_visual_inertial_pnp(ba, probs, initial_radius=r0)
    assert xs.shape == (len(probs), 16) and len(sums) == len(probs)
    for d, xg, sg in zip(probs, xs, sums):
        _check_oracle(d, xg, sg, r0)
        assert sg['solve_seconds'] == sums[0]['solve_seconds'] > 0


def test_batch_equals_single_calls_beyond_one_wave(ba):
    seeds = [_problem(synth.EUROC if k % 2 else synth.TUMVI, k % 4 != 3, 150 if k % 3 else 60, 900 + k)
             for k in range(16)]
    singles = [_single(ba, d) for d in seeds]
    n = 1600                          # more than 4 CTAs on each of the H100's 132 SMs
    xs, sums = pnp.batch_visual_inertial_pnp(ba, [seeds[i % 16] for i in range(n)])
    worst_cost, worst_state = 0.0, 0.0
    for i in range(n):
        d, (x1, s1) = seeds[i % 16], singles[i % 16]
        sg = sums[i]
        for k in ("iterations", "accepted_steps", "termination", "usable"):
            assert sg[k] == s1[k], (i, k)
        cost = max(abs(sg['final_cost'] - s1['final_cost']) / s1['final_cost'],
                   abs(sg['initial_cost'] - s1['initial_cost']) / s1['initial_cost'])
        state = np.linalg.norm(xs[i] - x1) / max(np.linalg.norm(x1 - d['frame']), 1e-3)
        worst_cost, worst_state = max(worst_cost, cost), max(worst_state, state)
        assert cost <= COST_TOL and state < STATE_TOL, (i, cost, state)
    print(f"batch of {n} vs single calls: largest relative cost difference {worst_cost:.3e}, "
          f"largest state difference {worst_state:.3e} x max(move, 1e-3)")


def test_launch_counts(ba):
    d = _problem(synth.EUROC, True, 150, 651)
    n0 = ba.kernel_launches
    _single(ba, d)
    assert ba.kernel_launches - n0 == 1
    for n in (1, 2, 300):
        n0 = ba.kernel_launches
        pnp.batch_visual_inertial_pnp(ba, [d] * n)
        assert ba.kernel_launches - n0 == 1
    n0 = ba.kernel_launches
    xs, sums = pnp.batch_visual_inertial_pnp(ba, [])
    assert ba.kernel_launches == n0 and xs.shape == (0, 16) and sums == []
    assert ba.lib.pvio_b200_batch_pnp_solve(ba.h, 0, None, None, 16, None, None) == 0


def _packed(probs):
    pbs, keep = (_lib.CPnpProblem * len(probs))(), []
    for pb, d in zip(pbs, probs):
        pnp._fill_problem(pb, keep, d['last'], d['imu'], d['pts'], d['zs'], d['cam_q'], d['cam_p'], d['imu_q'],
                          d['imu_p'], d['W'], d['use_inertial'], 1.0)
    return pbs, keep


def _spoil_n(pb):
    pb.n_points = -1


def _spoil_imu(pb):
    pb.use_inertial, pb.imu_data = 1, None


def _spoil_points(pb):
    pb.points = None


def _spoil_last(pb):
    pb.last_frame = None


@pytest.mark.parametrize("spoil", [_spoil_n, _spoil_imu, _spoil_points, _spoil_last, None],
                         ids=["negative_n_points", "inertial_without_imu", "null_points", "null_last_frame",
                              "short_stride"])
def test_rejections_leave_everything_untouched(ba, spoil):
    probs = [_problem(synth.EUROC, True, 40, 950 + k) for k in range(7)]
    pbs, keep = _packed(probs)
    stride = 16
    if spoil is None:
        stride = 15
    else:
        spoil(pbs[3])
    frames = np.full((7, 16), 12345.0)
    sms = (_lib.CSummary * 7)()
    opt = _lib.COptions(10, 1e6, 1, 0, 0.0)
    rc = ba.lib.pvio_b200_batch_pnp_solve(ba.h, 7, pbs, _lib.ptr(frames), stride, C.byref(opt), sms)
    assert rc == EINVAL
    assert np.all(frames == 12345.0)
    assert all(sms[i].iterations == 0 for i in range(7))
    xs, sums = pnp.batch_visual_inertial_pnp(ba, probs)            # the handle is still usable
    x1, s1 = _single(ba, probs[3])
    assert sums[3]['iterations'] == s1['iterations']
    assert np.linalg.norm(xs[3] - x1) < STATE_TOL * max(np.linalg.norm(x1 - probs[3]['frame']), 1e-3)


def test_buffer_growth_strided_frames_no_summaries():
    b = BundleAdjustor(max_windows=1, max_frames=4, max_landmarks=16, max_obs=64)
    try:
        small = [_problem(synth.EUROC, True, 8, 960 + k) for k in range(3)]
        xs, sums = pnp.batch_visual_inertial_pnp(b, small)
        for d, xg, sg in zip(small, xs, sums):
            _check_oracle(d, xg, sg, 0.0)
        large = [_problem(synth.TUMVI if k % 2 else synth.EUROC, k % 5 != 4, 400, 970 + k) for k in range(40)]
        pbs, keep = _packed(large)
        stride = 21
        frames = np.full((len(large), stride), -7.0)
        for i, d in enumerate(large):
            frames[i, :16] = d['frame']
        opt = _lib.COptions(10, 1e6, 1, 0, 0.0)
        rc = b.lib.pvio_b200_batch_pnp_solve(b.h, len(large), pbs, _lib.ptr(frames), stride,
                                             C.byref(opt), None)
        assert rc == 0
        assert np.all(frames[:, 16:] == -7.0)                       # the padding of each row is not touched
        for d, xg in zip(large, frames[:, :16]):
            xr, _ = _oracle(d, 0.0)
            assert np.linalg.norm(xg - xr) < STATE_TOL * max(np.linalg.norm(xr - d['frame']), 1e-3)
        d = _problem(synth.EUROC, True, 150, 651)
        x1, s1 = _single(b, d)
        _check_oracle(d, x1, s1, 0.0)
    finally:
        b.close()
