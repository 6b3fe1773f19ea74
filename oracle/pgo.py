"""oracle/pgo.py - CPU restatement of PL-SLAM's loop-closure pose-graph optimisation.  TEST INFRASTRUCTURE ONLY (see
oracle/__init__.py).

Follows MapHandler::loopClosureOptimizationCovGraphG2O, src/mapHandler.cpp:4185-4410 (called from both loop-closure
paths, :1028 and :3001): the graph of :4198-4290 (cov_graph_lists), g2o's computeInitialGuess() and optimize(maxItersPGO)
(initial_guess, optimize), and the write-back of :4298-4398 (cov_graph_write_back).  plf_pose_graph (csrc/pgo.cu) is
checked against optimize().

[UPSTREAM-RECALL] g2o is not on disk.  What follows restates from g2o's public sources the semantics the reference relies
on, as SURVEY Appendix A does for stvo-pl:
  VertexSE3 / EdgeSE3.  Poses are isometries X = (R, t).  The MQT vector of an isometry is (t; q_x, q_y, q_z), q the
    unit quaternion of R (Eigen's Quaternion(Matrix3), normalised) with the sign making w >= 0.  oplus(d): X <- X Inc(d),
    Inc(d) = (R(q), d_t) with q = (sqrt(1 - |d_q|^2), d_q), the identity rotation when 1 - |d_q|^2 < 0.  The error of an
    edge with measurement Z from vertex 0 (X_i) to vertex 1 (X_j) is e = MQT(Z^-1 (X_i^-1 X_j)), its chi2 e^T e (the
    information is the identity); H gets J_i^T J_i, J_j^T J_j and J_i^T J_j on the free vertices' blocks and b gets
    -J^T e.  A fixed vertex has no rows; an edge between two fixed vertices adds to chi2 only.  The Jacobians at d = 0
    (E = (R_E, t_E), q_E = (w, v), w >= 0):
        J_j = [R_E 0; 0 wI + [v]x],   J_i = [-R_Z^T  2 [t_E + R_Z^T t_Z]x R_Z^T; 0  (-wI + [v]x) R_Z^T]
    (tests/test_pgo_oracle.py pins them against central differences of error()).
  computeInitialGuess(): Dijkstra with unit edge cost from the fixed vertices; every reached free vertex is overwritten
    through its tree edge by parent Z (parent = vertex 0) or parent Z^-1.  With unit costs and strict relaxation this is
    a FIFO breadth-first search; the start vertices go in ascending id and a vertex's edges are visited in g2o's
    std::set<Edge*> order, which is pointer order and implementation-defined: DEFINED here as the order the edges are
    given (the reference's creation order).  Vertices without edges are inactive in g2o and never touched.
  OptimizationAlgorithmLevenberg::solve, per iteration (lambda = lambda_init at iteration 0, ni = 2):
        chi = chi2(X); build H, b at X
        repeat (trial): solve (H + lambda I) x = b (failure: chi_t = DBL_MAX); X_t = X (+) x; chi_t = chi2(X_t)
            rho = (chi - chi_t) / (sum x (lambda x + b) + 1e-3)
            rho > 0 and chi_t finite: lambda *= max(1/3, min(2/3, 1 - (2 rho - 1)^3)); ni = 2; X = X_t; chi = chi_t
            else: lambda *= ni; ni *= 2
        until not (rho < 0 and trials < 10)
        stop when trials == 10, rho == 0 or lambda is not finite; else the next iteration, up to max_iters.
    SparseOptimizer::optimize returns at once when no free vertex has edges.

Deviations from the reference (DESIGN.md §8): the log/exp round trips of :4242-4246, :4269-4270, :4286-4287,
:4303-4307 are not reproduced (the identity to rounding, except g2o's first-order SE3Quat::exp below theta = 1e-5,
off by less than 1e-10); g2o's re-orthogonalisation after 1000 oplus calls cannot be reached at 100 iterations x 10
trials and is not reproduced; a non-positive or non-finite pivot of the LDL^T stands in for cholmod's failure; a
component with edges but no fixed vertex is refused by plf_pose_graph (the reference never builds one).
"""
import math

import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

DBL_MAX = float(np.finfo(np.float64).max)
STOP = ("max_iters", "trials", "rho_zero", "lambda")
DENSE_MAX_N = 192   # solve() factors densely up to n = 6 n_free = 192 (32 free vertices), with splu beyond


# ---- isometries [..., 4, 4], the operation order of csrc/pgo.cu ---------------------------------------------------
def iso_mul(A, B):
    A, B = np.broadcast_arrays(np.asarray(A, np.float64), np.asarray(B, np.float64))
    C = np.zeros(A.shape)
    for r in range(3):
        for c in range(3):
            C[..., r, c] = A[..., r, 0] * B[..., 0, c] + A[..., r, 1] * B[..., 1, c] + A[..., r, 2] * B[..., 2, c]
        C[..., r, 3] = A[..., r, 0] * B[..., 0, 3] + A[..., r, 1] * B[..., 1, 3] + A[..., r, 2] * B[..., 2, 3] + A[..., r, 3]
    C[..., 3, 3] = 1.0
    return C


def iso_inv(A):
    A = np.asarray(A, np.float64)
    B = np.zeros(A.shape)
    for r in range(3):
        for c in range(3):
            B[..., r, c] = A[..., c, r]
        B[..., r, 3] = -(A[..., 0, r] * A[..., 0, 3] + A[..., 1, r] * A[..., 1, 3] + A[..., 2, r] * A[..., 2, 3])
    B[..., 3, 3] = 1.0
    return B


def quat(T):
    """(w, x, y, z) [..., 4] of the rotation block: Eigen's Quaternion(Matrix3), normalised, w >= 0"""
    T = np.asarray(T, np.float64)
    R = lambda i, j: T[..., i, j]
    tr = R(0, 0) + R(1, 1) + R(2, 2)
    with np.errstate(invalid="ignore", divide="ignore"):
        cases = []
        t = np.sqrt(tr + 1.0); h = 0.5 / t
        cases.append((0.5 * t, (R(2, 1) - R(1, 2)) * h, (R(0, 2) - R(2, 0)) * h, (R(1, 0) - R(0, 1)) * h))
        t = np.sqrt(R(2, 2) - R(0, 0) - R(1, 1) + 1.0); h = 0.5 / t                       # i = 2
        cases.append(((R(1, 0) - R(0, 1)) * h, (R(0, 2) + R(2, 0)) * h, (R(1, 2) + R(2, 1)) * h, 0.5 * t))
        t = np.sqrt(R(1, 1) - R(2, 2) - R(0, 0) + 1.0); h = 0.5 / t                       # i = 1
        cases.append(((R(0, 2) - R(2, 0)) * h, (R(0, 1) + R(1, 0)) * h, 0.5 * t, (R(2, 1) + R(1, 2)) * h))
        t = np.sqrt(R(0, 0) - R(1, 1) - R(2, 2) + 1.0); h = 0.5 / t                       # i = 0
        cases.append(((R(2, 1) - R(1, 2)) * h, 0.5 * t, (R(1, 0) + R(0, 1)) * h, (R(2, 0) + R(0, 2)) * h))
        sel = np.where(tr > 0.0, 0, np.where(R(2, 2) > np.where(R(1, 1) > R(0, 0), R(1, 1), R(0, 0)), 1,
                                              np.where(R(1, 1) > R(0, 0), 2, 3)))
        q = [np.choose(sel, [c[m] for c in cases]) for m in range(4)]
        n = np.sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3])
        s = np.where(q[0] / n < 0.0, -1.0 / n, 1.0 / n)
    return np.stack([q[0] * s, q[1] * s, q[2] * s, q[3] * s], -1)


def mqt(T):
    """(t; q_x, q_y, q_z) [..., 6]"""
    T = np.asarray(T, np.float64)
    return np.concatenate([T[..., :3, 3], quat(T)[..., 1:]], -1)


def quat_rot(w, v):
    """Eigen's Quaternion::toRotationMatrix for (w, v [..., 3])"""
    x, y, z = v[..., 0], v[..., 1], v[..., 2]
    tx, ty, tz = 2.0 * x, 2.0 * y, 2.0 * z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz, tyy, tyz, tzz = tx * x, ty * x, tz * x, ty * y, tz * y, tz * z
    return np.stack([np.stack([1.0 - (tyy + tzz), txy - twz, txz + twy], -1),
                     np.stack([txy + twz, 1.0 - (txx + tzz), tyz - twx], -1),
                     np.stack([txz - twy, tyz + twx, 1.0 - (txx + tyy)], -1)], -2)


def inc(d):
    """Inc(d) [..., 4, 4] of increments d [..., 6]: the inverse of mqt() on |d_q| <= 1, the identity rotation beyond"""
    d = np.asarray(d, np.float64)
    v = d[..., 3:]
    w2 = 1.0 - (v[..., 0] * v[..., 0] + v[..., 1] * v[..., 1] + v[..., 2] * v[..., 2])
    R = quat_rot(np.sqrt(np.maximum(w2, 0.0)), v)
    R = np.where((w2 < 0.0)[..., None, None], np.eye(3), R)
    T = np.zeros(d.shape[:-1] + (4, 4))
    T[..., :3, :3], T[..., :3, 3], T[..., 3, 3] = R, d[..., :3], 1.0
    return T


def oplus(X, d):
    return iso_mul(X, inc(d))


def error(Xi, Xj, Z):
    """e = MQT(Z^-1 (X_i^-1 X_j)) [..., 6]"""
    return mqt(iso_mul(iso_inv(Z), iso_mul(iso_inv(Xi), Xj)))


def jacobians(Xi, Xj, Z):
    """(e, J_i, J_j) at d = 0: rows are error components, columns increment components"""
    Z = np.asarray(Z, np.float64)
    E = iso_mul(iso_inv(Z), iso_mul(iso_inv(Xi), Xj))
    q = quat(E)
    e = np.concatenate([E[..., :3, 3], q[..., 1:]], -1)
    w, v = q[..., 0], q[..., 1:]
    sh = E.shape[:-2]
    Vx = np.zeros(sh + (3, 3))
    Vx[..., 0, 1], Vx[..., 0, 2], Vx[..., 1, 2] = -v[..., 2], v[..., 1], -v[..., 0]
    Vx -= np.swapaxes(Vx, -1, -2)
    I = np.eye(3)
    RZt = np.swapaxes(Z[..., :3, :3], -1, -2)
    p = E[..., :3, 3] + np.einsum("...ij,...j->...i", RZt, Z[..., :3, 3])
    P2 = np.zeros(sh + (3, 3))
    P2[..., 0, 1], P2[..., 0, 2], P2[..., 1, 2] = -2.0 * p[..., 2], 2.0 * p[..., 1], -2.0 * p[..., 0]
    P2 -= np.swapaxes(P2, -1, -2)
    Jj = np.zeros(sh + (6, 6))
    Jj[..., :3, :3] = E[..., :3, :3]
    Jj[..., 3:, 3:] = w[..., None, None] * I + Vx
    Ji = np.zeros(sh + (6, 6))
    Ji[..., :3, :3] = -RZt
    Ji[..., :3, 3:] = P2 @ RZt
    Ji[..., 3:, 3:] = (-w[..., None, None] * I + Vx) @ RZt
    return e, Ji, Jj


# ---- the graph ------------------------------------------------------------------------------------------------------
def _arrays(prob):
    T = np.asarray(prob["T"], np.float64).reshape(-1, 4, 4)
    fixed = np.asarray(prob["fixed"]).astype(bool).ravel()
    frm = np.asarray(prob["from"], np.int64).ravel()
    to = np.asarray(prob["to"], np.int64).ravel()
    Z = np.asarray(prob["Z"], np.float64).reshape(-1, 4, 4)
    return T, fixed, frm, to, Z


def initial_guess(T, fixed, frm, to, Z):
    """computeInitialGuess(): breadth-first from the fixed vertices (ascending id), each vertex's edges in the order
    given; returns the new estimates (unreached and fixed vertices keep theirs, bit for bit)"""
    X = np.array(T, np.float64, copy=True)
    adj = [[] for _ in range(len(X))]
    for k, (a, b) in enumerate(zip(frm, to)):
        adj[a].append(k)
        adj[b].append(k)
    seen = np.array(fixed, bool, copy=True)
    queue = [v for v in range(len(X)) if fixed[v]]
    h = 0
    while h < len(queue):
        v = queue[h]
        h += 1
        for k in adj[v]:
            u = to[k] if frm[k] == v else frm[k]
            if seen[u]:
                continue
            seen[u] = True
            X[u] = iso_mul(X[v], Z[k]) if frm[k] == v else iso_mul(X[v], iso_inv(Z[k]))
            queue.append(u)
    return X


def chi2(X, frm, to, Z):
    if not len(frm):
        return 0.0
    e = error(X[frm], X[to], Z)
    return float(np.sum(np.sum(e * e, 1)))


def free_index(fixed, frm, to):
    """the system block of each vertex: the free vertices with edges in id order, -1 for the others"""
    deg = np.bincount(np.concatenate([frm, to]).astype(np.int64), minlength=len(fixed))
    fidx = np.full(len(fixed), -1, np.int64)
    act = (~fixed) & (deg > 0)
    fidx[act] = np.arange(int(act.sum()))
    return fidx


def system(e, Ji, Jj, fi, fj, nf):
    """H (scipy.sparse CSC, symmetric) and b = -sum J^T e over the free vertices' blocks"""
    rows, cols, vals = [], [], []
    b = np.zeros(6 * nf)
    r6, c6 = np.meshgrid(np.arange(6), np.arange(6), indexing="ij")

    def put(m, ra, ca, L, R):
        blk = np.einsum("nki,nkj->nij", L[m], R[m])
        rows.append((6 * ra[m][:, None, None] + r6).ravel())
        cols.append((6 * ca[m][:, None, None] + c6).ravel())
        vals.append(blk.ravel())

    mi, mj = fi >= 0, fj >= 0
    put(mi, fi, fi, Ji, Ji)
    put(mj, fj, fj, Jj, Jj)
    both = mi & mj
    put(both, fi, fj, Ji, Jj)
    put(both, fj, fi, Jj, Ji)
    np.add.at(b, 6 * fi[mi][:, None] + np.arange(6), -np.einsum("nki,nk->ni", Ji[mi], e[mi]))
    np.add.at(b, 6 * fj[mj][:, None] + np.arange(6), -np.einsum("nki,nk->ni", Jj[mj], e[mj]))
    H = sp.coo_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(6 * nf, 6 * nf))
    return H.tocsc(), b


def ldlt_dense(A):
    """LDL^T without pivoting (the factorisation plf_pose_graph runs): (L with D on the diagonal, ok)"""
    A = np.array(A, np.float64, copy=True)
    n = len(A)
    ok = True
    for j in range(n):
        d = A[j, j]
        ok &= bool(d > 0.0 and d <= DBL_MAX)
        A[j + 1:, j] /= d
        A[j + 1:, j + 1:] -= np.outer(A[j + 1:, j], A[j + 1:, j] * d)
    return np.tril(A), ok


def solve(H, lam, b, solver="auto"):
    """(H + lam I) x = b: (x, ok).  dense: ldlt_dense and the two substitutions.  sparse: scipy splu on a symmetric
    fill-reducing ordering without row pivoting (diag_pivot_thresh = 0), so U's diagonal holds the pivots of an LDL^T
    of the symmetrically permuted matrix; they are all positive exactly when the matrix is positive definite, which is
    when the device's unpermuted LDL^T has positive pivots too.  ok = every pivot positive and finite."""
    n = H.shape[0]
    if solver == "dense" or (solver == "auto" and n <= DENSE_MAX_N):
        with np.errstate(all="ignore"):
            L, ok = ldlt_dense(H.toarray() + lam * np.eye(n))
            D = np.diag(L).copy()
            Lu = np.tril(L, -1) + np.eye(n)
            y = np.linalg.solve(Lu, b) if n else b
            x = np.linalg.solve(Lu.T, y / D) if n else b
        return x, ok
    try:
        lu = spla.splu((H + lam * sp.identity(n, format="csc")).tocsc(), permc_spec="MMD_AT_PLUS_A",
                       diag_pivot_thresh=0.0, options=dict(SymmetricMode=True))
    except RuntimeError:
        return np.full(n, np.nan), False
    with np.errstate(all="ignore"):
        x = lu.solve(b)
    D = lu.U.diagonal()
    return x, bool(np.all((D > 0.0) & (D <= DBL_MAX)) and np.all(np.isfinite(x)))


def lm_trials(chi, lam, ni, trial, it=0, trace=None):
    """One OptimizationAlgorithmLevenberg::solve: trial(lam) -> (chi_t, sum x (lam x + b), ok, state).  Returns
    (chi, lam, ni, trials, rho, state of the last accepted trial or None)"""
    trials, accepted_state = 0, None
    while True:
        chi_t, scale, ok, state = trial(lam)
        if not ok:
            chi_t = DBL_MAX
        with np.errstate(all="ignore"):
            rho = float(np.float64(chi - chi_t) / np.float64(scale + 1e-3))
        accept = rho > 0.0 and math.isfinite(chi_t)
        if trace is not None:
            trace.append(dict(iter=it, accepted=int(accept), lambda_=lam, chi=chi, chi_t=chi_t, rho=rho))
        if accept:
            lam *= max(1.0 / 3.0, min(1.0 - math.pow(2.0 * rho - 1.0, 3), 2.0 / 3.0))
            ni = 2.0
            chi = chi_t
            accepted_state = state
        else:
            lam *= ni
            ni *= 2.0   # a double in g2o (_ni)
        trials += 1
        if not (rho < 0.0 and trials < 10):
            return chi, lam, ni, trials, rho, accepted_state


def stop_reason(trials, rho, lam):
    """the iteration's verdict: None to go on, else the STOP name"""
    if trials == 10:
        return "trials"
    if rho == 0.0:
        return "rho_zero"
    if not math.isfinite(lam):
        return "lambda"
    return None


def optimize(prob, max_iters=100, lambda_init=1e-10, solver="auto", guess=True):
    """computeInitialGuess() then optimize(max_iters); prob in plf_pose_graph's layout.  Returns the binding's dict
    (T, iters, stop, trials, chi2_init, chi2, lambda_, trace as a list of dicts).  guess=False starts from prob's T
    as it is (the tests use it to permute the edges without changing the start)."""
    T, fixed, frm, to, Z = _arrays(prob)
    X = initial_guess(T, fixed, frm, to, Z) if guess else T.copy()
    chi = chi2(X, frm, to, Z)
    out = dict(chi2_init=chi, iters=0, stop="max_iters", trials=0, trace=[])
    fidx = free_index(fixed, frm, to)
    nf = int((fidx >= 0).sum())
    lam, ni = lambda_init, 2.0
    fi, fj = fidx[frm], fidx[to]
    for it in range(max_iters if nf else 0):
        e, Ji, Jj = jacobians(X[frm], X[to], Z)
        H, b = system(e, Ji, Jj, fi, fj, nf)

        def trial(lam_):
            x, ok = solve(H, lam_, b, solver)
            Xt = X.copy()
            free = np.nonzero(fidx >= 0)[0]
            Xt[free] = oplus(X[free], x.reshape(-1, 6)[fidx[free]])
            with np.errstate(all="ignore"):
                scale = float(np.sum(x * (lam_ * x + b)))
            return chi2(Xt, frm, to, Z), scale, ok, Xt

        chi, lam, ni, trials, rho, Xa = lm_trials(chi, lam, ni, trial, it, out["trace"])
        if Xa is not None:
            X = Xa
        out["iters"] = it + 1
        out["trials"] += trials
        s = stop_reason(trials, rho, lam)
        if s:
            out["stop"] = s
            break
    out.update(T=X, chi2=chi, lambda_=lam)
    return out


# ---- the reference's graph and write-back ---------------------------------------------------------------------------
def cov_graph_lists(full_graph, live, T_kf_w, lc_idx, lc_pose, min_ess=150, min_cov=75):
    """:4198-4290: the vertices are the live keyframes 0 .. kf_curr_idx (kf_curr_idx = the largest lc_idx[k][1];
    kf_prev_idx is forced to 0, :4208), keyframe 0 fixed; kf2kf edges for every live pair i < j <= kf_curr_idx with
    full_graph[i][j] >= min_ess or >= min_cov or |i - j| == 1 on the raw indices, in (i asc, j asc) order, measuring
    T_i^-1 T_j of the current poses; then one edge per loop closure lc_idx[k][0] -> [1] in list order, measuring
    expmap_se3(lc_pose[k]).  Returns plf_pose_graph's layout plus kf_list (the keyframe id of each vertex)."""
    from oracle import clib
    live = np.asarray(live, bool)
    T_kf_w = np.asarray(T_kf_w, np.float64)
    kf_curr = max(int(l[1]) for l in lc_idx)
    kf_list = [i for i in range(0, kf_curr + 1) if live[i]]
    pos = {k: n for n, k in enumerate(kf_list)}
    frm, to, Z = [], [], []
    for i in kf_list:
        for j in kf_list:
            if j > i and (full_graph[i][j] >= min_ess or full_graph[i][j] >= min_cov or abs(i - j) == 1):
                frm.append(pos[i]); to.append(pos[j])
                Z.append(iso_mul(iso_inv(T_kf_w[i]), T_kf_w[j]))
    for (a, b), x in zip([(int(l[0]), int(l[1])) for l in lc_idx], lc_pose):
        frm.append(pos[a]); to.append(pos[b])
        Z.append(np.asarray(clib.expmap_se3(np.asarray(x, np.float64)), np.float64))
    fixed = np.array([k == 0 for k in kf_list], np.uint8)
    return dict(kf_list=kf_list, T=T_kf_w[kf_list].copy(), fixed=fixed, **{"from": np.array(frm, np.int32)},
                to=np.array(to, np.int32), Z=np.array(Z, np.float64).reshape(-1, 4, 4))


def _xf(C, p):
    """Tkfw_corr.block(0,0,3,3) * p + Tkfw_corr.block(0,3,3,1)"""
    return C[:3, :3] @ np.asarray(p, np.float64) + C[:3, 3]


def cov_graph_write_back(T_kf_w, live, kf_list, T_opt, points, lines, points_kf_idx, lines_kf_idx):
    """:4298-4398 as written.  T_kf_w [n_kf, 4, 4] with live[i] = map_keyframes[i] != NULL; T_opt: the optimised pose of
    each keyframe of kf_list; points / lines: per map index None (deleted) or dict(point3D [3] / line3D [6],
    med_obs_dir [3], dir_list [m, 3]); *_kf_idx: per keyframe the landmarks anchored there (map_points_kf_idx).
    Every keyframe of kf_list takes its pose and Tkfw_corr = T_new T_prev^-1 moves its landmarks (point3D, both ends of
    line3D, med_obs_dir and each dir_list entry, all like points); every keyframe after kf_curr_idx, and its landmarks,
    then takes the last Tkfw_corr.  The reference does not check those keyframes for NULL (:4357): one raises here.
    Returns (T_kf_w, points, lines), new copies."""
    T = np.array(T_kf_w, np.float64, copy=True)
    pts = [None if p is None else {k: np.array(v, np.float64, copy=True) for k, v in p.items()} for p in points]
    lns = [None if p is None else {k: np.array(v, np.float64, copy=True) for k, v in p.items()} for p in lines]

    def move(kf, C):
        for i in points_kf_idx[kf]:
            if pts[i] is not None:
                pts[i]["point3D"] = _xf(C, pts[i]["point3D"])
                pts[i]["med_obs_dir"] = _xf(C, pts[i]["med_obs_dir"])
                pts[i]["dir_list"] = np.array([_xf(C, d) for d in pts[i]["dir_list"]]).reshape(-1, 3)
        for i in lines_kf_idx[kf]:
            if lns[i] is not None:
                L = lns[i]["line3D"]
                lns[i]["line3D"] = np.concatenate([_xf(C, L[:3]), _xf(C, L[3:])])
                lns[i]["med_obs_dir"] = _xf(C, lns[i]["med_obs_dir"])
                lns[i]["dir_list"] = np.array([_xf(C, d) for d in lns[i]["dir_list"]]).reshape(-1, 3)

    C = None
    for kf, Tn in zip(kf_list, np.asarray(T_opt, np.float64).reshape(-1, 4, 4)):
        C = Tn @ iso_inv(T[kf])
        T[kf] = Tn
        move(kf, C)
    for i in range(max(kf_list) + 1, len(T)):
        if not live[i]:
            raise ValueError(f"keyframe {i} after kf_curr_idx is NULL: the reference dereferences it (:4357)")
        T[i] = C @ T[i]
        move(i, C)
    return T, pts, lns
