// Trust-region control of the solve, ON THE DEVICE: the minimiser logic of ceres::Solve as PVIO configures it
// (estimation/ceres/solver_options.h:26-33: SPARSE_SCHUR, DOGLEG -> TRADITIONAL_DOGLEG, Jacobi scaling, function
// tolerance 1e-6, gradient tolerance 1e-10, parameter tolerance 1e-8, initial radius 1e4; Ceres 1.14
// trust_region_minimizer.cc / dogleg_strategy.cc), one decision record (WinCtrl) per window.
//
// One iteration is a FIXED kernel sequence (api.cu: iteration_body), every kernel looks at its window's flags first:
//   lin_obs (state)            FIRST body only (the window has no linearisation yet): into the window's buffer set WinCtrl::buf
//   schur, solve               skipped when the previous step was rejected (`reuse`: same linearisation, same GN step)
//   backsub  (+ tr_after_backsub)   GN step of the inverse depths; is the GN step inside the trust region?
//   jv_vision, jv_aux (+ tr_after_jv)   only when it is not: |J v|^2 for the Cauchy point, dogleg interpolation
//   candidate                  Plus(x, step)
//   lin_obs (candidate)        (a body skipped because its linear solve failed, mu * 10: the STATE again, with the new mu)
//                              the FULL linearisation of the candidate into the other buffer set: its cost is the
//                              reprojection cost the decision needs; on acceptance the buffer sets swap, so the
//                              residual-only evaluation of ceres and the relinearisation after it are one sweep
//   aux_cost (+ tr_decide)     IMU / prior / plane cost at the candidate; accept / reject, radius, mu, termination
// so a whole solve is max_iterations identical bodies captured in ONE CUDA graph: no device -> host read, no host
// decision, one launch per solve (single window) or per batch (per-window termination).
#pragma once
#include "ba_types.h"
#include "../../include/pvio_b200.h"

namespace pvio {

__device__ __forceinline__ double global_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return (double)t;
}

__device__ __forceinline__ void tr_terminate(WinCtrl &c, int termination) { c.termination = termination; c.done = 1; }

// After the back-substitution (acc[1..3, 5, 7, 8] hold the landmark parts of the step scalars).
// Mirrors the top of the trust-region iteration: gradient tolerance at a fresh linearisation, the retry of a
// failed linear solve with a larger mu (dogleg_strategy.cc), iteration count, the trust-region test of the GN step.
__device__ inline void tr_after_backsub(WinCtrl &c, const double *acc) {
    c.skip = 0; c.need_jv = 0;
    if (c.fresh) {
        if (c.iteration == 0 && c.accepted == 0) c.initial_cost = c.cost;
        if (c.gmax <= 1e-10) { tr_terminate(c, PVIO_B200_TERM_CONVERGENCE); return; }
    }
    if (c.max_time_ns > 0.0 && global_ns() - c.t_start_ns > c.max_time_ns) { c.done = 1; return; }
    if (c.iteration >= c.max_iter) { c.done = 1; return; }
    if (c.solve_failed) {
        c.mu *= 10.0; c.reuse = 0; c.skip = 1; c.have_lin = 0;      // the pivots depend on mu: linearise the state again
        if (c.mu > 1.0) { c.usable = 0; tr_terminate(c, PVIO_B200_TERM_FAILURE); }
        return;
    }
    ++c.iteration;
    const double gn_norm = sqrt(c.gn_norm2 + acc[3]);
    c.step_a = 0.0; c.step_b = 1.0; c.step_norm = gn_norm;
    if (gn_norm > c.radius) c.need_jv = 1;
}

// After the J.v sweeps (acc[9], acc[10] = |J v|^2 of the vision / other blocks): DoglegStrategy::ComputeStep
// (TRADITIONAL_DOGLEG), all norms in the diag-scaled space; then the model cost change of the chosen step.
__device__ inline void tr_after_jv(WinCtrl &c, const double *acc) {
    if (c.done || c.skip) return;
    const double gdx = c.g_dot_dx + acc[1];                  // g . dx_gn
    const double rdx = c.dx_reg_dx + acc[2];                 // dx_gn^T (mu D) dx_gn
    double sa = 0.0, sb = 1.0, grad2 = 0.0, v_rd = 0.0, jv2 = 0.0;
    if (c.need_jv) {
        const double gn_norm = c.step_norm, radius = c.radius;
        grad2 = c.grad2 + acc[7];
        v_rd = c.v_reg_dx + acc[8];
        jv2 = acc[9] + acc[10];
        const double g_norm = sqrt(grad2);
        const double alpha = grad2 / jv2;
        if (g_norm * alpha >= radius) {                       // scaled steepest descent to the boundary
            sa = radius / g_norm; sb = 0.0;
        } else {                                              // dogleg interpolation (dogleg_strategy.cc)
            const double b_dot_a = -alpha * gdx;
            const double a2 = (alpha * g_norm) * (alpha * g_norm);
            const double bma2 = a2 - 2.0 * b_dot_a + gn_norm * gn_norm;
            const double cc = b_dot_a - a2;
            const double dd = sqrt(cc * cc + bma2 * (radius * radius - a2));
            const double beta = cc <= 0 ? (dd - cc) / bma2 : (radius * radius - a2) / (dd + cc);
            sa = alpha * (1.0 - beta); sb = beta;
        }
        c.step_norm = radius;
    }
    c.step_a = sa; c.step_b = sb;
    // model cost change -(g.s + s^T H s / 2) of s = sb dx_gn - sa v, using H dx_gn = -g - (mu D) dx_gn
    const double dHd = -gdx - rdx, vHd = -grad2 - v_rd;
    const double sHs = sb * sb * dHd - 2.0 * sa * sb * vHd + sa * sa * jv2;
    c.model_change = -(sb * gdx - sa * grad2) - 0.5 * sHs;
    if (!(c.model_change > 0.0)) { c.radius *= 0.5; c.reuse = 1; c.skip = 1; c.fresh = 0; }      // invalid step
}

// After the candidate sweeps: step acceptance (trust_region_minimizer.cc).  Returns true when the candidate
// becomes the state (the caller copies it).
__device__ inline bool tr_decide(WinCtrl &c, const double *acc, double cand_vis, double aux_cost) {
    c.fresh = 0;
    if (c.done || c.skip) return false;
    c.cand_cost_vis = cand_vis;
    c.cand_cost = cand_vis + aux_cost;
    const double cost = c.cost;
    const double x_norm = sqrt(c.xnorm2 + acc[5]);
    const double step_amb = sqrt(acc[6] + acc[4]);
    if (step_amb <= 1e-8 * (x_norm + 1e-8)) { tr_terminate(c, PVIO_B200_TERM_CONVERGENCE); return false; }
    if (fabs(cost - c.cand_cost) <= 1e-6 * cost) { tr_terminate(c, PVIO_B200_TERM_CONVERGENCE); return false; }
    const double rel = (cost - c.cand_cost) / c.model_change;
    bool accept = false;
    if (rel > 1e-3) {
        accept = true;
        ++c.accepted;
        c.cost = c.cand_cost;                // re-evaluated by the next linearisation, as ceres does at the accepted point
        if (rel < 0.25) c.radius *= 0.5;
        if (rel > 0.75) c.radius = fmax(c.radius, 3.0 * c.step_norm);
        c.mu = fmax(1e-8, 2.0 * c.mu / 10.0);
        c.reuse = 0;
    } else {
        c.radius *= 0.5;
        c.reuse = 1;
    }
    if (c.radius <= 1e-32) tr_terminate(c, PVIO_B200_TERM_CONVERGENCE);
    // iteration budget spent: after a REJECTED step nothing is left to do; after an accepted one ceres still evaluates
    // cost, gradient and Jacobian at the new point (final_cost is that re-evaluated cost -- with the aliased bias
    // linearisation point of quirk Q1 it differs from the candidate cost), which the next body's linearisation does
    // before tr_after_backsub stops the window
    else if (c.iteration >= c.max_iter && !accept) c.done = 1;
    return accept;
}

// named (may be NULL): a window with named[w] == 0 is only marked finished, so that every kernel of the loop skips it
static __global__ void init_ctrl_kernel(WinCtrl *ctrl, double mu, double radius, int max_iter, double max_time_s, int w0,
                                        const uint8_t *named = nullptr) {
    WinCtrl &c = ctrl[blockIdx.x + w0];
    if (named && !named[blockIdx.x + w0]) { if (threadIdx.x == 0) c.done = 1; return; }
    if (threadIdx.x == 0) {
        c.mu = mu; c.radius = radius; c.iteration = 0; c.accepted = 0; c.done = 0;
        c.termination = PVIO_B200_TERM_NO_CONVERGENCE; c.solve_failed = 0; c.have_scale = 0; c.usable = 1;
        c.reuse = 0; c.need_jv = 0; c.skip = 0; c.fresh = 0; c.max_iter = max_iter; c.buf = 0; c.have_lin = 0;
        c.step_a = 0.0; c.step_b = 1.0; c.step_norm = 0.0; c.initial_cost = 0.0; c.cost = 0.0; c.cand_cost = 0.0;
        c.max_time_ns = max_time_s > 0.0 && max_time_s < 1e5 ? max_time_s * 1e9 : 0.0;
        c.t_start_ns = global_ns();
    }
}

}  // namespace pvio
