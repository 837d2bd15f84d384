"""ORACLE (test infrastructure) -- the dogleg trust-region strategy of Ceres (<= 2.1 DoglegStrategy, TRADITIONAL_DOGLEG
and SUBSPACE_DOGLEG) on the pose-graph problem of oracle/posegraph.py.

PARITY UNPINNED, like oracle/posegraph.py: Ceres is not available, so this is a restatement of the published algorithm
(DESIGN.md §4 "Dogleg"), not a transcript.  The problem, Jacobi scaling, step evaluator, tolerance tests, invalid-step
counter and minimum-cost iterate are those of oracle/posegraph.py; only the strategy differs.  The Gauss-Newton solves are
exact (SciPy SuperLU), the subspace basis is a column-pivoted Householder QR (scipy.linalg.qr) and the quartic of the
subspace boundary minimiser is solved with numpy.roots.

The LM oracle itself is not touched: `solve` with trust_region_strategy="lm" (the default) calls oracle.posegraph.solve.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import scipy.linalg as sla
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from oracle import posegraph as PG

MIN_MU, MAX_MU, MU_INCREASE = 1e-8, 1.0, 10.0
KKT_COSINE = 0.99


@dataclass
class Options(PG.Options):
    trust_region_strategy: str = "lm"     # "lm" | "dogleg"  (ceres_trust_strategy, solvers/ceres_solver.cpp:46-58)
    dogleg_type: str = "traditional"      # "traditional" | "subspace"  (ceres_dogleg_type, :138-155)


@dataclass
class Summary(PG.Summary):
    linear_solves: int = 0                # Gauss-Newton / LM linear solves, retries at a larger mu included


def traditional_step(g_s, gn_s, alpha, radius):
    """ComputeTraditionalDoglegStep in the scaled space: returns (s_s, step_norm)."""
    gn_norm = float(np.linalg.norm(gn_s))
    if gn_norm <= radius:
        return gn_s.copy(), gn_norm
    g_norm = float(np.linalg.norm(g_s))
    if alpha * g_norm >= radius:
        return -(radius / g_norm) * g_s, radius
    a, b = -alpha * g_s, gn_s
    b_dot_a = float(b @ a)
    a_sq = float(a @ a)
    bma_sq = a_sq - 2.0 * b_dot_a + float(b @ b)
    c = b_dot_a - a_sq
    d = np.sqrt(c * c + bma_sq * (radius * radius - a_sq))
    beta = (d - c) / bma_sq if c <= 0 else (radius * radius - a_sq) / (d + c)
    s = (1.0 - beta) * a + beta * b
    return s, float(np.linalg.norm(s))


def boundary_polynomial(g, B, r):
    """Quartic in the Lagrange multiplier y whose roots give the stationary points of 1/2 x^T B x + g^T x on ||x|| = r,
    coefficients from the highest power down."""
    tr = B[0, 0] + B[1, 1]
    det = B[0, 0] * B[1, 1] - B[0, 1] * B[1, 0]
    adj = np.array([[B[1, 1], -B[0, 1]], [-B[1, 0], B[0, 0]]])
    ag = adj @ g
    r2 = r * r
    return np.array([r2, 2.0 * r2 * tr, r2 * (tr * tr + 2.0 * det) - g @ g, -2.0 * (g @ ag - r2 * det * tr),
                     r2 * det * det - ag @ ag])


def boundary_minimum(g, B, r, roots=np.roots):
    """The subspace boundary minimiser: the lowest model value over the real parts of the quartic's roots, each projected
    onto ||x|| = r.  None when no root gives a usable point or when the first-order (KKT) check fails."""
    best, best_f = None, np.inf
    for y in np.real(roots(boundary_polynomial(g, B, r))):
        try:
            x = -np.linalg.solve(B + y * np.eye(2), g)
        except np.linalg.LinAlgError:
            continue
        n = float(np.linalg.norm(x))
        if not np.isfinite(n) or n <= 0.0:
            continue
        x = (r / n) * x
        f = 0.5 * float(x @ B @ x) + float(g @ x)
        if f < best_f:
            best, best_f = x, f
    if best is None:
        return None
    grad = B @ best + g
    cosine = -float(best @ grad) / (float(np.linalg.norm(best)) * float(np.linalg.norm(grad)))
    if cosine < KKT_COSINE:
        return None
    return best


def subspace_basis(g_s, gn_s):
    """Orthonormal basis of span{g_s, gn_s} by column-pivoted QR; rank 1 when |R22| <= 2 eps |R11|."""
    Q, R, _ = sla.qr(np.column_stack([g_s, gn_s]), mode="economic", pivoting=True)
    rank1 = abs(R[1, 1]) <= 2.0 * np.finfo(np.float64).eps * abs(R[0, 0])
    return Q[:, :1] if rank1 else Q[:, :2], rank1


def subspace_step(g_s, gn_s, alpha, radius, basis, rank1, g2, B2, roots=np.roots):
    """ComputeSubspaceDoglegStep: returns (s_s, step_norm)."""
    gn_norm = float(np.linalg.norm(gn_s))
    if gn_norm <= radius:
        return gn_s.copy(), gn_norm
    if rank1:
        return -(radius / float(np.linalg.norm(g_s))) * g_s, radius
    x = boundary_minimum(g2, B2, radius, roots)
    if x is None:
        return traditional_step(g_s, gn_s, alpha, radius)
    return basis @ x, radius


def solve(poses, edge_a, edge_b, z, cov=None, U=None, fixed=0, opts: Options | None = None):
    """oracle.posegraph.solve with the trust-region strategy of `opts`.  Returns (optimised poses, Summary)."""
    o = opts or Options()
    if o.trust_region_strategy == "lm":
        base = PG.Options(**{k: getattr(o, k) for k in PG.Options.__dataclass_fields__})
        x, s = PG.solve(poses, edge_a, edge_b, z, cov=cov, U=U, fixed=fixed, opts=base)
        return x, Summary(**vars(s), linear_solves=s.iterations)   # LM runs one linear solve per iteration
    if o.trust_region_strategy != "dogleg" or o.dogleg_type not in ("traditional", "subspace"):
        raise ValueError((o.trust_region_strategy, o.dogleg_type))
    subspace = o.dogleg_type == "subspace"
    x = np.array(poses, dtype=np.float64)
    if U is None:
        U = np.stack([PG.sqrt_information(c) for c in cov])
    pb = PG.Problem(x, edge_a, edge_b, z, U, fixed, o.loss_function, o.loss_scale)
    sm = Summary()
    nfree = 3 * len(pb.free)
    if nfree == 0 or len(pb.ea) == 0:
        sm.termination = "CONVERGENCE (nothing to optimise)"
        return x, sm

    def evaluate(xx):
        return pb.cost(xx), pb.residuals(xx)

    def grad_and_jac(xx, r, scale):
        J = pb.jacobian(xx)
        g = J.T @ r
        if o.jacobi_scaling:
            if scale is None:
                scale = 1.0 / (1.0 + np.sqrt(np.asarray(J.multiply(J).sum(axis=0)).reshape(-1)))
            J = J @ sp.diags(scale)
        elif scale is None:
            scale = np.ones(nfree)
        xs = pb.params(xx)
        proj = pb.params(pb.plus(xx, -g))
        gmax = float(np.max(np.abs(xs - proj))) if len(xs) else 0.0
        return J, scale, gmax

    cost, r = evaluate(x)
    sm.initial_cost = cost
    J, scale, gmax = grad_and_jac(x, r, None)
    x_norm = float(np.linalg.norm(pb.params(x)))
    best_x, minimum_cost = x.copy(), cost

    # DoglegStrategy state
    radius, mu, reuse = o.initial_trust_region_radius, MIN_MU, False
    D = g_s = gn_s = None
    alpha = 0.0
    basis = g2 = B2 = None
    rank1 = False
    # TrustRegionStepEvaluator state
    max_nonmono = o.max_consecutive_nonmonotonic_steps if o.use_nonmonotonic_steps else 0
    ev_min = ev_cur = ev_ref = ev_cand = cost
    acc_ref = acc_cand = 0.0
    n_nonmono = 0
    invalid_steps = 0
    it = 0
    step_successful = False
    sm.trace.append((0, cost, True, radius))
    converged_at_start = gmax <= o.gradient_tolerance
    if converged_at_start:
        sm.termination = "CONVERGENCE (gradient tolerance)"
    while not converged_at_start:
        if it >= o.max_num_iterations:
            sm.termination = "NO_CONVERGENCE (max iterations)"
            break
        if step_successful and gmax <= o.gradient_tolerance:
            sm.termination = "CONVERGENCE (gradient tolerance)"
            break
        if radius <= o.min_trust_region_radius:
            sm.termination = "CONVERGENCE (min trust region radius)"
            break
        it += 1
        step_successful = False
        # DoglegStrategy::ComputeStep
        ok = True
        if not reuse:
            D = np.sqrt(np.clip(np.asarray(J.multiply(J).sum(axis=0)).reshape(-1), o.min_lm_diagonal, o.max_lm_diagonal))
            rhs = J.T @ r
            g_s = rhs / D
            Jg = J @ (g_s / D)
            alpha = float(g_s @ g_s) / float(Jg @ Jg)
            ok = False
            while mu < MAX_MU:   # ComputeGaussNewtonStep: (J^T J + mu D^2) y = J^T r, mu grows on failure
                sm.linear_solves += 1
                try:
                    y = spla.splu((J.T @ J + sp.diags(mu * D * D)).tocsc()).solve(rhs)
                    ok = bool(np.all(np.isfinite(y)))
                except RuntimeError:
                    ok = False
                if ok:
                    break
                mu *= MU_INCREASE
            if ok:
                gn_s = -D * y
                if subspace:
                    basis, rank1 = subspace_basis(g_s, gn_s)
                    JB = J @ (basis / D[:, None])
                    g2, B2 = basis.T @ g_s, JB.T @ JB
                reuse = True
        valid = False
        if ok:
            if subspace:
                s_s, step_norm = subspace_step(g_s, gn_s, alpha, radius, basis, rank1, g2, B2)
            else:
                s_s, step_norm = traditional_step(g_s, gn_s, alpha, radius)
            step = s_s / D
            mr = J @ step
            model_cost_change = -float(mr @ (r + mr / 2.0))
            valid = model_cost_change > 0.0
        if not valid:   # DoglegStrategy::StepIsInvalid
            invalid_steps += 1
            if invalid_steps >= o.max_num_consecutive_invalid_steps:
                sm.termination = "FAILURE (too many invalid steps)"
                sm.usable = False
                break
            mu *= MU_INCREASE
            reuse = False
            sm.trace.append((it, cost, False, radius))
            continue
        invalid_steps = 0
        delta = step * scale
        cand = pb.plus(x, delta)
        cand_cost, cand_r = evaluate(cand)
        step_norm_x = float(np.linalg.norm(pb.params(x) - pb.params(cand)))
        if step_norm_x <= o.parameter_tolerance * (x_norm + o.parameter_tolerance):
            sm.termination = "CONVERGENCE (parameter tolerance)"
            break
        cost_change = cost - cand_cost
        if abs(cost_change) <= o.function_tolerance * cost:
            sm.termination = "CONVERGENCE (function tolerance)"
            break
        rel = (ev_cur - cand_cost) / model_cost_change
        hist = (ev_ref - cand_cost) / (acc_ref + model_cost_change)
        quality = max(rel, hist)
        if quality > o.min_relative_decrease:
            x, cost, r = cand, cand_cost, cand_r
            x_norm = float(np.linalg.norm(pb.params(x)))
            J, scale, gmax = grad_and_jac(x, r, scale)
            step_successful = True
            sm.successful_steps += 1
            # DoglegStrategy::StepAccepted (no clamp to max_trust_region_radius, DESIGN.md §4)
            if quality < 0.25:
                radius *= 0.5
            if quality > 0.75:
                radius = max(radius, 3.0 * step_norm)
            mu = max(MIN_MU, mu / 5.0)
            reuse = False
            ev_cur = cost
            acc_cand += model_cost_change
            acc_ref += model_cost_change
            if ev_cur < ev_min:
                ev_min = ev_cur; n_nonmono = 0; ev_cand = ev_cur; acc_cand = 0.0
            else:
                n_nonmono += 1
                if ev_cur > ev_cand:
                    ev_cand = ev_cur; acc_cand = 0.0
            if n_nonmono == max_nonmono:
                ev_ref = ev_cand; acc_ref = acc_cand
            if cost < minimum_cost:
                minimum_cost, best_x = cost, x.copy()
        else:   # DoglegStrategy::StepRejected: shrink, keep the Gauss-Newton step
            radius *= 0.5
            reuse = True
        sm.trace.append((it, cost, step_successful, radius))
    sm.iterations = it
    sm.final_cost = minimum_cost
    return (best_x if sm.usable else np.array(poses, dtype=np.float64)), sm
