"""CPU restatement (float64 numpy) of the camera fit with shared intrinsics (DESIGN.md section 1, "Shared intrinsics"): images in
one group keep their own roll and pitch and share s = ln f_rel (and cx_rel, cy_rel with principal_point).  The residuals, cost,
start and normalisation are oracle_calib's; the step solves the group's dense damped joint system by np.linalg.cholesky, so
the GPU's Schur-complement algebra (csrc/calib.cuh, fit_group_step_kernel) is checked by an independent route.

Joint parameters of a group with kept members i_1 < ... < i_m: (r_1, e_1, ..., r_m, e_m, s[, cx_rel, cy_rel]).
"""
import math

import numpy as np

import oracle_calib as oc


def _image_theta(x, j, K):
    """Image j's theta (P entries) from the joint parameter vector."""
    return np.concatenate([x[2 * j:2 * j + 2], x[len(x) - K:]])


def _evaluate(x, members, fields, P, huber):
    """(C_G, joint A, joint g, per-member C_i) at x; the sum over members in their index order."""
    K = P - 2
    m = len(members)
    N = 2 * m + K
    A = np.zeros((N, N))
    g = np.zeros(N)
    C = 0.0
    Ci = []
    for j, i in enumerate(members):
        up, lat, mask = fields[i]
        c, a, gi, _ = oc.evaluate(_image_theta(x, j, K), up, lat, mask, P, huber)
        idx = np.r_[2 * j, 2 * j + 1, np.arange(2 * m, N)]
        A[np.ix_(idx, idx)] += a
        g[idx] += gi
        C += c
        Ci.append(c)
    return C, A, g, Ci


def _solve(M, b):
    """M x = b by Cholesky (np.linalg.cholesky); None when M is not positive definite."""
    try:
        L = np.linalg.cholesky(M)
    except np.linalg.LinAlgError:
        return None
    return np.linalg.solve(L.T, np.linalg.solve(L, b))


def group_start(fields, members, principal_point=False, inits=None):
    """({i: image i's own start theta, 5 entries}, the group's shared start (s, cx_rel, cy_rel): the mean in index order)."""
    starts = {}
    for i in members:
        up, lat, mask = fields[i]
        init = None if inits is None else inits[i]
        if init is None:
            starts[i] = list(oc.start(up, lat, mask)) + [0.0, 0.0]
        else:
            starts[i] = [init[0], init[1], math.log(init[2]), init[3] if principal_point else 0.0, init[4] if principal_point else 0.0]
    shared = []
    for k in range(3):
        t = starts[members[0]][2 + k]
        for i in members[1:]:
            t += starts[i][2 + k]
        shared.append(t / len(members))
    return starts, shared


def fit_group(fields, members, principal_point=False, huber=None, max_iterations=50, inits=None):
    """One group: fields[i] = (up [H, W, 2], latitude [H, W] degrees, mask or None) for i in members (index order); inits[i] as
    oracle_calib.fit's init, or None.  Returns {i: dict(theta, params, cost, iterations, status)} with oracle_calib.fit's keys."""
    P = 5 if principal_point else 3
    K = P - 2
    starts, shared = group_start(fields, members, principal_point, inits)
    nan = {"theta": [math.nan] * 5, "params": [math.nan] * 5, "cost": math.nan, "iterations": 1, "status": 2}
    # the first evaluation: drop members without 2 residuals or with a zero on their roll / pitch diagonal
    kept, count = [], 0
    for i in members:
        up, lat, mask = fields[i]
        _, a, _, cnt = oc.evaluate(np.array(starts[i][:2] + shared[:K]), up, lat, mask, P, huber)
        if cnt < 2 or a[0, 0] == 0 or a[1, 1] == 0:
            continue
        kept.append(i)
        count += cnt
    x = np.array([v for i in kept for v in starts[i][:2]] + shared[:K], np.float64)
    if kept:
        C, A, g, Ci = _evaluate(x, kept, fields, P, huber)
    if not kept or count < 2 * len(kept) + K or np.any(np.diag(A)[2 * len(kept):] == 0):
        return {i: dict(nan) for i in members}
    evals = 1
    lam = oc.LAMBDA0
    status = None
    while status is None:
        delta = None
        while lam <= oc.LAMBDA_MAX:
            delta = _solve(A + lam * np.diag(np.diag(A)), -g)
            if delta is not None:
                break
            lam *= 10.0
        if delta is None:
            status = 0
            break
        if np.all(np.abs(delta) <= oc.STEP_RTOL * (1.0 + np.abs(x))):
            status = 0
            break
        if evals >= max_iterations:
            status = 1
            break
        cand = x + delta
        Cc, Ac, gc, Cic = _evaluate(cand, kept, fields, P, huber)
        evals += 1
        if Cc < C:
            done = C - Cc <= oc.COST_RTOL * C
            x, C, A, g, Ci = cand, Cc, Ac, gc, Cic
            lam /= 10.0
            if done:
                status = 0
        else:
            lam *= 10.0
            if lam > oc.LAMBDA_MAX:
                status = 0
    out = {}
    for i in members:
        if i not in kept:
            out[i] = dict(nan, iterations=evals)
            continue
        j = kept.index(i)
        full = oc.normalise(list(_image_theta(x, j, K)) + [0.0] * (5 - P))
        params = [math.degrees(full[0]), math.degrees(full[1]), math.exp(full[2]), full[3], full[4]]
        out[i] = {"theta": full, "params": params, "cost": Ci[j], "iterations": evals, "status": status}
    return out


def fit_groups(ups, lats, masks, groups, principal_point=False, huber=None, max_iterations=50, inits=None):
    """calibrate.fit_camera(..., groups=groups) restated: a list of per-image results (oracle_calib.fit's keys)."""
    members = {}
    for i, gid in enumerate(groups):
        members.setdefault(gid, []).append(i)
    fields = [(u, l, None if masks is None else masks[i]) for i, (u, l) in enumerate(zip(ups, lats))]
    out = [None] * len(ups)
    for mem in members.values():
        for i, r in fit_group(fields, mem, principal_point, huber, max_iterations, inits).items():
            out[i] = r
    return out


def joint_residuals(x, members, fields, P):
    """The group's residual vector and Jacobian at joint parameters x (for scipy.optimize.least_squares)."""
    K = P - 2
    m = len(members)
    rs, Js = [], []
    for j, i in enumerate(members):
        up, lat, mask = fields[i]
        ru, Ju, rl, Jl = oc.residuals(_image_theta(x, j, K), up, lat, mask, P)
        J = np.concatenate([Ju, Jl])
        full = np.zeros((J.shape[0], 2 * m + K))
        full[:, 2 * j:2 * j + 2] = J[:, :2]
        full[:, 2 * m:] = J[:, 2:]
        rs.append(np.concatenate([ru, rl]))
        Js.append(full)
    return np.concatenate(rs), np.concatenate(Js)
