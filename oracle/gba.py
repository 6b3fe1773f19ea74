"""oracle/gba.py - CPU restatement of PL-SLAM's global bundle adjustment.  TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

Follows MapHandler::levMarquardtOptimizationGBA, src/mapHandler.cpp:2101-2699, called from
MapHandler::globalBundleAdjustment :1995-2099 with X = [x_kf_w of every keyframe but keyframe 0 | point3D of every point |
line3D of every line] and one Vector6i per observation (plf_lba_problem's layout, see plf_global_ba):
  first pass on the map's values :2117-2356 (point rows :2119-2225, line rows :2227-2353), initial lambda :2358-2365,
  H_ii += lambda H_ii and SimplicialLDLT solve :2366-2375, update T = expmap(X) * inverse(expmap(DX)) / X += DX
  :2376-2385, LM iterations :2390-2672 (point rows :2400-2504, line rows :2506-2632, normalise :2635, stop tests
  :2637, :2667, lambda schedule and step :2648-2665), write-back :2673-2697.
The rows are numpy-vectorised restatements of the same expressions as oracle/lba.c (the reference's GBA rows are
LBA's rows).  H is assembled as a scipy.sparse matrix from the lower triangle the reference's writes leave, which is all
SimplicialLDLT reads (Eigen's default UpLo = Lower), and solved with scipy.sparse.linalg.splu: no dense N x N matrix,
so maps of hundreds of keyframes fit.

What the reference does that looks unintended, and what happens here (ref_quirks = 1 reproduces it, 0 = the evident intent):
  (g1) :2115 `double err` is not initialised before the first pass accumulates into it, and :2356 divides it by
       Npt_obs + Nls_obs, two counters never incremented.  Defined here as starting at 0, so err = sum / 0 (+inf, or NaN
       for a zero sum).  Intent: start at 0, divide by the number of observations.
  (g2) :2359 `int Hmax`: each diagonal entry d is compared with the int (`d > Hmax || d < -Hmax`) and stored truncated
       (`Hmax = fabs(d)`), so a maximum below 1 gives lambda = 0 (an undamped first step).  A value >= 2^31 does not
       fit an int; the conversion is undefined in C++ and defined here as what x86-64 cvttsd2si yields (the reference is
       built -march=native on x86-64): INT_MIN, whose negation wraps to INT_MIN.  Intent: the double maximum.
  (g3) :2635 the LM iterations divide by the same zero counters: err = +inf (NaN at 0), so the stop test :2637 never
       fires, `err > err_prev` is never true and every step is applied with lambda *= lambda_k; the loop ends at
       max_iters or at |DX| < min_error_change.  Intent: divide by the number of observations.
  (g4) :2520-2521 the LM line rows read both end points from one block of X at stride 3 (as LBA's q2).  Intent: the
       landmark's own 6 values.
  (g5) :2523 the LM line rows take the map's pose of the observing keyframe (as LBA's q3); unlike LBA they clamp with
       SlamConfig::homogTh().  Intent: the pose in X.
  (g6) :2349-2350 the first pass writes the line/keyframe coupling as H(idx+i, jdx+j) += Hij(i,j) and
       H(jdx+j, idx+i) += Hij(i,j) with Hij = w J_L J_T^T, so the lower triangle (landmark row x pose column) holds
       w J_T J_L^T.  The LM iterations write it correctly (:2629).  Intent: w J_L J_T^T.
"""
import math

import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from oracle import clib

DBL_EPSILON = float(np.finfo(np.float64).eps)
INT_MIN = -2 ** 31


def opts(lambda_=1e-5, lambda_k=10.0, max_iters=15, homog_th=1e-7, min_error=DBL_EPSILON, min_error_change=DBL_EPSILON,
         ref_quirks=1):
    """SlamConfig::lambdaLbaLM / lambdaLbaK / maxItersLba (:2116, :2391) and the DBL_EPSILON literals (:2637, :2667)."""
    return dict(lambda_=lambda_, lambda_k=lambda_k, max_iters=max_iters, homog_th=homog_th, min_error=min_error,
                min_error_change=min_error_change, ref_quirks=ref_quirks)


def _xform(Ti, P):
    """Tiw.block(0,0,3,3) * P + Tiw.block(0,3,3,1), per row, summed left to right as oracle/lba.c does"""
    return np.stack([Ti[:, r, 0] * P[:, 0] + Ti[:, r, 1] * P[:, 1] + Ti[:, r, 2] * P[:, 2] + Ti[:, r, 3] for r in range(3)], 1)


def _jac_pose(gz2, fxdx, fydy, gx, gy, gz):
    return np.stack([+gz2 * fxdx * gz, +gz2 * fydy * gz, -gz2 * (fxdx * gx + fydy * gy),
                     -gz2 * (fxdx * gx * gy + fydy * gy * gy + fydy * gz * gz),
                     +gz2 * (fxdx * gx * gx + fxdx * gz * gz + fydy * gx * gy),
                     +gz2 * (fydy * gx * gz - fxdx * gy * gz)], 1)


def _jac_lm(gz2, fxdx, fydy, gx, gy, gz, Ti):
    """J3^T * R, out_j = v0 R_0j + v1 R_1j + v2 R_2j"""
    v = [+gz2 * fxdx * gz, +gz2 * fydy * gz, -gz2 * (fxdx * gx + fydy * gy)]
    return np.stack([v[0] * Ti[:, 0, j] + v[1] * Ti[:, 1, j] + v[2] * Ti[:, 2, j] for j in range(3)], 1)


def point_rows(cam, homog, Ti, Xw, xy):
    """:2133-2175 / :2410-2449: residual norm, Cauchy weight, J wrt the pose (6) and the point (3)"""
    Xwi = _xform(Ti, Xw)
    px = cam["cx"] + cam["fx"] * Xwi[:, 0] / Xwi[:, 2]
    py = cam["cy"] + cam["fy"] * Xwi[:, 1] / Xwi[:, 2]
    dx, dy = xy[:, 0] - px, xy[:, 1] - py
    nrm = np.sqrt(dx * dx + dy * dy)
    gx, gy, gz = Xwi[:, 0], Xwi[:, 1], Xwi[:, 2]
    gz2 = 1.0 / np.maximum(homog, gz * gz)
    fxdx, fydy = cam["fx"] * dx, cam["fy"] * dy
    den = np.maximum(homog, nrm)[:, None]
    JT = _jac_pose(gz2, fxdx, fydy, gx, gy, gz) / den
    JX = _jac_lm(gz2, fxdx, fydy, gx, gy, gz, Ti) / den
    return nrm, 1.0 / (1.0 + nrm * nrm), JT, JX


def line_rows(cam, homog, Ti, P, Q, le):
    """:2241-2318 / :2518-2590: residual norm, Cauchy weight, J wrt the pose (6) and the two end points (6)"""
    Pwi, Qwi = _xform(Ti, P), _xform(Ti, Q)
    prj = lambda W: (cam["cx"] + cam["fx"] * W[:, 0] / W[:, 2], cam["cy"] + cam["fy"] * W[:, 1] / W[:, 2])
    (ppx, ppy), (qpx, qpy) = prj(Pwi), prj(Qwi)
    e0 = le[:, 0] * ppx + le[:, 1] * ppy + le[:, 2]
    e1 = le[:, 0] * qpx + le[:, 1] * qpy + le[:, 2]
    nrm = np.sqrt(e0 * e0 + e1 * e1)
    fxlx, fyly = cam["fx"] * e0, cam["fy"] * e1   # the two residuals, as the reference writes it (:2261-2262)
    den = np.maximum(homog, nrm)
    out = []
    for W, e in ((Pwi, e0), (Qwi, e1)):
        gx, gy, gz = W[:, 0], W[:, 1], W[:, 2]
        gz2 = 1.0 / np.maximum(homog, gz * gz)
        out.append((_jac_pose(gz2, fxlx, fyly, gx, gy, gz), _jac_lm(gz2, fxlx, fyly, gx, gy, gz, Ti) * (e / den)[:, None]))
    (JP, JPw), (JQ, JQw) = out
    JT = (JP * e0[:, None] + JQ * e1[:, None]) / den[:, None]
    return nrm, 1.0 / (1.0 + nrm * nrm), JT, np.concatenate([JPw, JQw], 1)


def _pose_inv(x):
    return clib.inverse_se3(clib.expmap_se3(x))


def normal_equations(cam, prob, X, T0inv, first, quirks, homog):
    """H (lower triangle, scipy.sparse CSC), g and the weighted error sum at X, as the reference's rows write them.
    first: the first pass (map poses and landmarks, (g6) coupling); else an LM iteration ((g4), (g5) when quirks)."""
    nkf, npt, nls = len(prob["kf_pose"]), len(prob["pt"]), len(prob["ls"])
    N = 6 * nkf + 3 * npt + 6 * nls
    fT = np.asarray(prob["fixed_T"], np.float64).reshape(-1, 4, 4)
    fTi = np.stack([clib.inverse_se3(T) for T in fT]) if len(fT) else np.zeros((0, 4, 4))
    Tcur = T0inv if first else (np.stack([_pose_inv(X[6 * i:6 * i + 6]) for i in range(nkf)]) if nkf else np.zeros((0, 4, 4)))

    def pose_of(kf, use_map):
        kf = np.asarray(kf)
        loc = np.clip(kf, 0, None)
        src = T0inv if use_map else Tcur
        Ti = src[loc] if nkf else np.zeros((len(kf), 4, 4))
        fixed = kf < 0
        if fixed.any():
            Ti[fixed] = fTi[-1 - kf[fixed]]
        return Ti

    rows, cols, vals = [], [], []
    g = np.zeros(N)
    err = 0.0

    def add(kf, jdx, dim, nrm, w, JT, JL, swap):
        nonlocal err
        loc = kf >= 0
        idx = 6 * kf
        np.add.at(g, jdx[:, None] + np.arange(dim), JL * (nrm * w)[:, None])
        np.add.at(g, (idx[loc, None] + np.arange(6)), JT[loc] * (nrm * w)[loc, None])
        err += float(np.sum(nrm * nrm * w))
        li, lj = np.tril_indices(dim)
        rows.append((jdx[:, None] + li).ravel()); cols.append((jdx[:, None] + lj).ravel())
        vals.append((JL[:, li] * JL[:, lj] * w[:, None]).ravel())
        pi, pj = np.tril_indices(6)
        rows.append((idx[loc, None] + pi).ravel()); cols.append((idx[loc, None] + pj).ravel())
        vals.append((JT[loc][:, pi] * JT[loc][:, pj] * w[loc, None]).ravel())
        a, b = np.meshgrid(np.arange(dim), np.arange(6), indexing="ij")
        a, b = a.ravel(), b.ravel()
        U, V = (JT, JL) if swap else (JL, JT)   # (g6): landmark row a carries J_T, pose column b carries J_L
        rows.append((jdx[loc, None] + a).ravel()); cols.append((idx[loc, None] + b).ravel())
        vals.append((U[loc][:, a] * V[loc][:, b] * w[loc, None]).ravel())

    po_lm, po_kf = np.asarray(prob["pt_obs_lm"]), np.asarray(prob["pt_obs_kf"])
    if len(po_lm):
        Xw = X[6 * nkf + 3 * po_lm[:, None] + np.arange(3)]
        nrm, w, JT, JX = point_rows(cam, homog, pose_of(po_kf, first), Xw, np.asarray(prob["pt_obs_xy"], np.float64).reshape(-1, 2))
        add(po_kf, 6 * nkf + 3 * po_lm, 3, nrm, w, JT, JX, False)
    lo_lm, lo_kf = np.asarray(prob["ls_obs_lm"]), np.asarray(prob["ls_obs_kf"])
    if len(lo_lm):
        base = 6 * nkf + 3 * npt
        if not first and quirks:
            P = Q = X[base + 3 * lo_lm[:, None] + np.arange(3)]                 # (g4)
        else:
            P = X[base + 6 * lo_lm[:, None] + np.arange(3)]
            Q = X[base + 6 * lo_lm[:, None] + 3 + np.arange(3)]
        Ti = pose_of(lo_kf, first or bool(quirks))                            # (g5)
        nrm, w, JT, JL = line_rows(cam, homog, Ti, P, Q, np.asarray(prob["ls_obs_le"], np.float64).reshape(-1, 3))
        add(lo_kf, base + 6 * lo_lm, 6, nrm, w, JT, JL, first and bool(quirks))
    r = np.concatenate(rows) if rows else np.zeros(0, int)
    c = np.concatenate(cols) if cols else np.zeros(0, int)
    v = np.concatenate(vals) if vals else np.zeros(0)
    return sp.coo_matrix((v, (r, c)), shape=(N, N)).tocsc(), g, err


def solve_lower(Hl, g):
    """SimplicialLDLT(H).solve(g) where only the lower triangle of H is read: the symmetric matrix tril + tril^T - diag"""
    Hs = (Hl + Hl.T - sp.diags(Hl.diagonal())).tocsc()
    return spla.splu(Hs).solve(g)


def cvttsd2si(v):
    """(int)v as x86-64 computes it: truncation toward zero, INT_MIN ("integer indefinite") outside int's range or NaN"""
    return int(v) if -2147483648.0 <= v < 2147483648.0 else INT_MIN


def hmax_int(diag):
    """(g2) :2359-2364 as written: `int Hmax = 0.0; if (d > Hmax || d < -Hmax) Hmax = fabs(d);` in index order"""
    h = 0
    for d in map(float, diag):
        neg = h if h == INT_MIN else -h   # -INT_MIN wraps
        if d > h or d < neg:
            h = cvttsd2si(abs(d))
    return float(h)


def zero_block_landmark(diag, nkf, npt):
    """The first landmark (points, then lines) whose block on the diagonal `diag` of the first pass has an exactly zero
    entry, else -1.  Such a problem is refused before any step, as oracle/lba.c and plf_global_ba refuse it."""
    lm = np.asarray(diag)[6 * nkf:]
    z = np.concatenate([(lm[:3 * npt].reshape(-1, 3) == 0).any(1), (lm[3 * npt:].reshape(-1, 6) == 0).any(1)])
    return int(np.argmax(z)) if z.any() else -1


def _apply(X, DX, nkf):
    Y = X.copy()
    for i in range(nkf):
        Tp = clib.expmap_se3(X[6 * i:6 * i + 6])
        Y[6 * i:6 * i + 6] = clib.logmap_se3(Tp @ clib.inverse_se3(clib.expmap_se3(DX[6 * i:6 * i + 6])))
    Y[6 * nkf:] += DX[6 * nkf:]
    return Y


def _div(a, b):
    with np.errstate(divide="ignore", invalid="ignore"):
        return float(np.float64(a) / np.float64(b))


def global_ba(cam, prob, o=None):
    """levMarquardtOptimizationGBA; prob as plf_global_ba takes it.  Returns clib.local_ba's dict (X split into
    kf_pose / pt / ls, the moved flags plf_global_ba also fills, iters, err, lambda_), or dict(rc=clib.LBA_ZERO_BLOCK,
    zero_lm) for a landmark whose first-pass block has a zero diagonal entry."""
    o = o or opts()
    q = bool(o["ref_quirks"])
    kf = np.asarray(prob["kf_pose"], np.float64).reshape(-1, 6)
    pt = np.asarray(prob["pt"], np.float64).reshape(-1, 3)
    ls = np.asarray(prob["ls"], np.float64).reshape(-1, 6)
    nkf, npt = len(kf), len(pt)
    nobs = len(prob["pt_obs_lm"]) + len(prob["ls_obs_lm"])
    X0 = np.concatenate([kf.ravel(), pt.ravel(), ls.ravel()])
    T0inv = np.stack([_pose_inv(x) for x in kf]) if nkf else np.zeros((0, 4, 4))
    homog = o["homog_th"]
    lam = o["lambda_"]
    # ---- first pass (:2117-2385)
    H, g, s = normal_equations(cam, prob, X0, T0inv, True, q, homog)
    err = _div(s, 0) if q else s / nobs                                          # (g1)
    dg = H.diagonal()
    zl = zero_block_landmark(dg, nkf, npt)
    if zl >= 0:
        return dict(rc=clib.LBA_ZERO_BLOCK, zero_lm=zl)
    lam *= hmax_int(dg) if q else float(np.max(np.abs(dg)))                      # (g2)
    H = H + sp.diags(lam * dg)
    DX = solve_lower(H, g)
    X = _apply(X0, DX, nkf)
    err_prev = err
    # ---- LM iterations (:2390-2672)
    iters = 1
    while iters < o["max_iters"]:
        H, g, s = normal_equations(cam, prob, X, T0inv, False, q, homog)
        err = _div(s, 0) if q else s / nobs                                      # (g3)
        if abs(err - err_prev) < o["min_error_change"] or err < o["min_error"]:
            break
        H = H + sp.diags(lam * H.diagonal())
        DX = solve_lower(H, g)
        if err > err_prev:
            lam /= o["lambda_k"]
        else:
            lam *= o["lambda_k"]
            X = _apply(X, DX, nkf)
        if math.sqrt(float(DX @ DX)) < o["min_error_change"]:
            break
        err_prev = err
        iters += 1
    d = X - X0
    nk, n3 = 6 * nkf, 3 * npt
    return dict(rc=0, kf_pose=X[:nk].reshape(-1, 6), pt=X[nk:nk + n3].reshape(-1, 3), ls=X[nk + n3:].reshape(-1, 6),
                pt_moved=np.sqrt((d[nk:nk + n3].reshape(-1, 3) ** 2).sum(1)) > 0.01,
                ls_moved=np.sqrt((d[nk + n3:].reshape(-1, 6) ** 2).sum(1)) > 0.01,
                iters=iters, err=err, lambda_=lam)
