"""CPU restatement (float64 numpy) of the camera-track fit (DESIGN.md section 1, "Camera tracks"): each group is one sequence of
evenly spaced frames in index order, with its own roll and pitch per frame and shared s = ln f_rel (and cx_rel, cy_rel with
principal_point).  The residuals, weights, start and normalisation are oracle_calib's (oracle_confidence's with weights); each
frame's cost is divided by its residual count M_t, and a random-walk prior ties neighbouring frames:

    C_S = sum_t C_t / M_t + 1/2 sum_t ((r_t+1 - r_t) / sigma_r)^2 + ((e_t+1 - e_t) / sigma_e)^2     (radians over degrees)

The step solves the damped joint system (A + lambda diag A) delta = -g directly: a dense np.linalg.cholesky, or for long
sequences LAPACK's banded Cholesky (scipy.linalg.cholesky_banded) of the locals' block with the shared unknowns eliminated
densely, so the GPU's chain recursion (csrc/calib.cuh, fit_seq_step_kernel) is checked by an independent route.

Joint parameters of a sequence of m frames: (r_1, e_1, ..., r_m, e_m, s[, cx_rel, cy_rel]).
"""
import math

import numpy as np
import scipy.sparse

import oracle_calib as oc
import oracle_confidence as ocf

DENSE_MAX = 400   # joint unknowns up to which the step uses the dense Cholesky


def _frame_theta(x, j, K):
    return np.concatenate([x[2 * j:2 * j + 2], x[len(x) - K:]])


def _weights(weights, i):
    return (None, None) if weights is None or weights[i] is None else weights[i]


def evaluate(x, members, fields, P, huber, wr, we, weights=None):
    """(C_S, joint A, joint g, each frame's own C_t, each frame's M_t) at x; the prior's terms included."""
    K = P - 2
    m = len(members)
    N = 2 * m + K
    rows, cols, vals = [], [], []   # A's entries, summed where they repeat
    g = np.zeros(N)
    C = 0.0
    Ct, Mt = [], []
    for j, i in enumerate(members):
        up, lat, mask = fields[i]
        wu, wl = _weights(weights, i)
        c, a, gi, cnt = ocf.evaluate(_frame_theta(x, j, K), up, lat, mask, P, huber, wu, wl)
        idx = np.r_[2 * j, 2 * j + 1, np.arange(2 * m, N)]
        if cnt > 0:
            rows.append(np.repeat(idx, P))
            cols.append(np.tile(idx, P))
            vals.append((a / cnt).ravel())
            g[idx] += gi / cnt
            C += c / cnt
        Ct.append(c)
        Mt.append(cnt)
    for t in range(m - 1):
        for k, w in ((0, wr), (1, we)):
            a, b = 2 * t + k, 2 * t + 2 + k
            d = x[b] - x[a]
            C += 0.5 * w * d * d
            rows.append(np.array([a, b, a, b]))
            cols.append(np.array([a, b, b, a]))
            vals.append(np.array([w, w, -w, -w]))
            g[a] -= w * d
            g[b] += w * d
    cat = lambda v, t: np.concatenate(v) if v else np.zeros(0, t)
    A = scipy.sparse.coo_matrix((cat(vals, float), (cat(rows, int), cat(cols, int))), shape=(N, N)).tocsr()
    return C, (A.toarray() if N <= DENSE_MAX else A), g, Ct, Mt


def _solve_dense(M, b):
    try:
        L = np.linalg.cholesky(M)
    except np.linalg.LinAlgError:
        return None
    return np.linalg.solve(L.T, np.linalg.solve(L, b))


def _solve_banded(M, b, K):
    """M x = b for the damped joint matrix: the locals' block (bandwidth 3) by scipy.linalg.cholesky_banded, the K shared
    unknowns by a dense Cholesky of their Schur complement; None when either is not positive definite."""
    import scipy.linalg as sl

    M = scipy.sparse.csr_matrix(M)
    n = M.shape[0] - K
    T = M[:n, :n]
    ab = np.zeros((4, n))
    for d in range(4):
        ab[3 - d, d:] = T.diagonal(d)
    try:
        cb = sl.cholesky_banded(ab)
    except np.linalg.LinAlgError:
        return None
    E = M[:n, n:].toarray()
    X = sl.cho_solve_banded((cb, False), np.column_stack([b[:n], E]))
    S = M[n:, n:].toarray() - E.T @ X[:, 1:]
    xs = _solve_dense(S, b[n:] - E.T @ X[:, 0])
    if xs is None:
        return None
    return np.concatenate([X[:, 0] - X[:, 1:] @ xs, xs])


def sequence_start(fields, members, principal_point=False, inits=None, weights=None):
    """The start: each frame's own (closed form or init), the shared entries the mean in index order, the rolls unwrapped along
    the sequence.  Returns the joint vector of 2 m + 3 entries (all three shared entries)."""
    starts = []
    for i in members:
        up, lat, mask = fields[i]
        init = None if inits is None else inits[i]
        if init is None:
            starts.append(list(ocf.start(up, lat, mask, *_weights(weights, i))) + [0.0, 0.0])
        else:
            starts.append([init[0], init[1], math.log(init[2]), init[3] if principal_point else 0.0, init[4] if principal_point else 0.0])
    shared = []
    for k in range(3):
        t = starts[0][2 + k]
        for s in starts[1:]:
            t += s[2 + k]
        shared.append(t / len(members))
    for j in range(1, len(starts)):
        r = starts[j][0]
        starts[j][0] = r - 2.0 * math.pi * np.rint((r - starts[j - 1][0]) / (2.0 * math.pi))
    return np.array([v for s in starts for v in s[:2]] + shared, np.float64)


def fit_sequence(fields, members, sigma, principal_point=False, huber=None, max_iterations=50, inits=None, weights=None):
    """One sequence: fields[i] = (up [H, W, 2], latitude [H, W] degrees, mask or None) for i in members (frame order); sigma =
    (sigma_roll, sigma_pitch) in degrees.  Returns {i: dict(theta, params, cost, iterations, status)} (oracle_calib.fit's
    keys; cost is the frame's own C_t)."""
    P = 5 if principal_point else 3
    K = P - 2
    wr, we = 1.0 / sigma[0] ** 2, 1.0 / sigma[1] ** 2
    m = len(members)
    x = sequence_start(fields, members, principal_point, inits, weights)[:2 * m + K]
    C, A, g, Ct, Mt = evaluate(x, members, fields, P, huber, wr, we, weights)
    evals = 1
    nan = {"theta": [math.nan] * 5, "params": [math.nan] * 5, "cost": math.nan, "iterations": 1, "status": 2}
    bad = sum(Mt) < 2 + K or np.any(A.diagonal()[2 * m:] == 0)
    if m == 1:
        bad = bad or A[0, 0] == 0 or A[1, 1] == 0
    if bad:
        return {i: dict(nan) for i in members}
    solve = _solve_dense if len(x) <= DENSE_MAX else (lambda M, b: _solve_banded(M, b, K))
    lam = oc.LAMBDA0
    status = None
    while status is None:
        delta = None
        while lam <= oc.LAMBDA_MAX:
            damp = lam * A.diagonal()
            delta = solve(A + (np.diag(damp) if isinstance(A, np.ndarray) else scipy.sparse.diags(damp)), -g)
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
        try:
            Cc, Ac, gc, Ctc, _ = evaluate(cand, members, fields, P, huber, wr, we, weights)
        except ZeroDivisionError:   # f_rel underflowed to 0: no cost (the kernel's is NaN), rejected
            Cc = math.inf
        evals += 1
        if Cc < C:
            done = C - Cc <= oc.COST_RTOL * C
            x, C, A, g, Ct = cand, Cc, Ac, gc, Ctc
            lam /= 10.0
            if done:
                status = 0
        else:
            lam *= 10.0
            if lam > oc.LAMBDA_MAX:
                status = 0
    out = {}
    for j, i in enumerate(members):
        full = oc.normalise(list(_frame_theta(x, j, K)) + [0.0] * (5 - P))
        params = [math.degrees(full[0]), math.degrees(full[1]), math.exp(full[2]), full[3], full[4]]
        out[i] = {"theta": full, "params": params, "cost": Ct[j], "iterations": evals, "status": status, "x": x}
    return out


def fit_sequences(ups, lats, masks, groups, sigma, principal_point=False, huber=None, max_iterations=50, inits=None, weights=None):
    """calibrate.fit_camera(..., groups=groups, smoothness=sigma) restated: a list of per-frame results."""
    sig = (float(sigma), float(sigma)) if np.isscalar(sigma) else tuple(float(v) for v in sigma)
    members = {}
    for i, gid in enumerate(groups):
        members.setdefault(gid, []).append(i)
    fields = [(u, l, None if masks is None else masks[i]) for i, (u, l) in enumerate(zip(ups, lats))]
    out = [None] * len(ups)
    for mem in members.values():
        for i, r in fit_sequence(fields, mem, sig, principal_point, huber, max_iterations, inits, weights).items():
            out[i] = r
    return out


def stacked_residuals(x, members, fields, P, sigma):
    """The residual vector whose half squared norm is C_S (least squares), its Jacobian, and per entry the frame's M_t (0 for
    the prior's entries): pixel residuals scaled by 1 / sqrt(M_t), then the prior's differences over sigma."""
    K = P - 2
    m = len(members)
    N = 2 * m + K
    rs, Js, Ms = [], [], []
    for j, i in enumerate(members):
        up, lat, mask = fields[i]
        ru, Ju, rl, Jl = oc.residuals(_frame_theta(x, j, K), up, lat, mask, P)
        r = np.concatenate([ru, rl])
        J = np.concatenate([Ju, Jl])
        full = np.zeros((J.shape[0], N))
        full[:, 2 * j:2 * j + 2] = J[:, :2]
        full[:, 2 * m:] = J[:, 2:]
        s = 1.0 / math.sqrt(r.size) if r.size else 0.0
        rs.append(r * s)
        Js.append(full * s)
        Ms.append(np.full(r.size, float(r.size)))
    for t in range(m - 1):
        for k in range(2):
            row = np.zeros((1, N))
            row[0, 2 * t + 2 + k], row[0, 2 * t + k] = 1.0 / sigma[k], -1.0 / sigma[k]
            rs.append(np.array([(x[2 * t + 2 + k] - x[2 * t + k]) / sigma[k]]))
            Js.append(row)
            Ms.append(np.zeros(1))
    return np.concatenate(rs), np.concatenate(Js), np.concatenate(Ms)
