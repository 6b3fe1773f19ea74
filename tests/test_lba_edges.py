"""CPU checks behind tests/test_lba_edges_gpu.py: the reference-shaped local maps (synth.local_map_problem), the maps that
put rows on the clamps and signs of the local BA's rows, the host-loop branch cases (read from the iteration trace of
oracle/lba.c), and the oracle's refusal of a landmark whose first-pass block has a zero diagonal entry.  The helpers here
build the maps the GPU file runs."""
import numpy as np
import pytest

import plslam_b200 as plf
from oracle import clib, gba
from plslam_b200 import synth

CAM = plf.KITTI_CAMERA


# ---- the maps ---------------------------------------------------------------------------------------------------------
def _proj(T, P):
    Ti = np.linalg.inv(T)
    Pc = Ti[:3, :3] @ P + Ti[:3, 3]
    return np.array([CAM["cx"] + CAM["fx"] * Pc[0] / Pc[2], CAM["cy"] + CAM["fy"] * Pc[1] / Pc[2]])


def _line_obs(T, P, Q, rng, noise=0.3):
    s = np.append(_proj(T, P) + noise * rng.standard_normal(2), 1.0)
    e = np.append(_proj(T, Q) + noise * rng.standard_normal(2), 1.0)
    le = np.cross(s, e)
    return le / np.hypot(le[0], le[1])


def _copy(p):
    return {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in p.items()}


def edge_map(homog_th, seed=11):
    """A local map (n_fixed = 3 from keyframe 0, the identity; 6 local keyframes) with five landmarks whose first pass
    has a row on an edge of k_lba_rows, each also observed by well-posed rows of fixed keyframes:
      point n   on keyframe 0's optical axis, observed there at (cx, cy): residual exactly 0 (nrm < homog_th)
      point n+1 on local keyframe 0's optical axis at depth sqrt(homog_th) / 2 (the depth clamp), observed there 316 px off
      point n+2 1 m behind local keyframe 0, observed by it at its (mirrored) projection: negative depth
      line 0    start point on local keyframe 0's optical axis at depth sqrt(homog_th) / 2; under (q2) the LM rows of
                line 0 read that point, so with homog_th above 1e-7 they reach the clamp only through (q4)'s literal
      line 1    in keyframe 0's plane x = 0, observed there as the line x = cx: both end-point residuals exactly 0
    The small-depth points sit on the optical axis so that the clamped rows do not set the damping of the whole map."""
    p = synth.local_map_problem(CAM, n_kf=6, n_fixed=3, seed=seed)
    rng = np.random.default_rng(seed + 100)
    T = p["truth"]["T"]
    assert np.array_equal(T[0], np.eye(4)) and np.array_equal(p["fixed_T"][0], np.eye(4))
    T0 = synth.expmap_se3(p["kf_pose"][0])   # local keyframe 0 as the first pass sees it
    d = 0.5 * np.sqrt(homog_th)
    local0 = lambda c: (T0 @ np.append(c, 1.0))[:3]
    q = _copy(p)
    A, B, Cn = np.array([0.0, 0.0, 12.0]), local0([0.0, 0.0, d]), local0([0.5, 0.3, -1.0])
    n = len(p["pt"])
    obs = [(n, -1, np.array([CAM["cx"], CAM["cy"]]))]
    obs += [(n, k, _proj(T[-1 - k], A) + 0.3 * rng.standard_normal(2)) for k in (-2, -3)]
    obs += [(n + 1, k, _proj(T[-1 - k], B) + 0.3 * rng.standard_normal(2)) for k in (-1, -2)]
    obs += [(n + 1, 0, np.array([CAM["cx"] + 300.0, CAM["cy"] + 100.0]))]
    obs += [(n + 2, k, _proj(T[-1 - k], Cn) + 0.3 * rng.standard_normal(2)) for k in (-1, -2)]
    obs += [(n + 2, 0, _proj(T0, Cn) + 0.3 * rng.standard_normal(2))]
    q["pt"] = np.concatenate([p["pt"], [A, B, Cn]])
    q["pt_obs_lm"] = np.concatenate([p["pt_obs_lm"], [o[0] for o in obs]]).astype(np.int32)
    q["pt_obs_kf"] = np.concatenate([p["pt_obs_kf"], [o[1] for o in obs]]).astype(np.int32)
    q["pt_obs_xy"] = np.concatenate([p["pt_obs_xy"], [o[2] for o in obs]])
    S, E = local0([0.0, 0.0, d]), local0([0.8, 0.3, 4.0])
    P1, Q1 = np.array([0.0, -1.0, 10.0]), np.array([0.0, 1.0, 12.0])
    lo = [(0, k, _line_obs(T[-1 - k], S, E, rng)) for k in (-1, -2)]
    lo += [(0, 0, np.array([1.0, 0.0, -(CAM["cx"] + 0.3)]))]   # 0.3 px from S's projection, 144 px from E's
    lo += [(1, -1, np.array([1.0, 0.0, -CAM["cx"]]))]
    lo += [(1, k, _line_obs(T[-1 - k], P1, Q1, rng)) for k in (-2, -3)]
    q["ls"] = np.concatenate([[np.concatenate([S, E]), np.concatenate([P1, Q1])], p["ls"]])
    q["ls_obs_lm"] = np.concatenate([[o[0] for o in lo], p["ls_obs_lm"] + 2]).astype(np.int32)
    q["ls_obs_kf"] = np.concatenate([[o[1] for o in lo], p["ls_obs_kf"]]).astype(np.int32)
    q["ls_obs_le"] = np.concatenate([[o[2] for o in lo], p["ls_obs_le"]]).reshape(-1, 3)
    return q


def zero_block_map(kind="pt"):
    """A local map plus one landmark seen once, by keyframe 0 (the identity), at its exact projection: every entry of its
    first-pass block is 0.  Returns (problem, index of that landmark among the points then the lines)."""
    p = synth.local_map_problem(CAM, n_kf=3, n_fixed=2, seed=1)
    assert np.array_equal(p["fixed_T"][0], np.eye(4))
    q = _copy(p)
    if kind == "pt":
        q["pt"] = np.concatenate([p["pt"], [[0.0, 0.0, 15.0]]])
        q["pt_obs_lm"] = np.append(p["pt_obs_lm"], len(p["pt"])).astype(np.int32)
        q["pt_obs_kf"] = np.append(p["pt_obs_kf"], -1).astype(np.int32)
        q["pt_obs_xy"] = np.concatenate([p["pt_obs_xy"], [[CAM["cx"], CAM["cy"]]]])
        return q, len(p["pt"])
    q["ls"] = np.concatenate([p["ls"], [[0.0, -1.0, 10.0, 0.0, 1.0, 12.0]]])
    q["ls_obs_lm"] = np.append(p["ls_obs_lm"], len(p["ls"])).astype(np.int32)
    q["ls_obs_kf"] = np.append(p["ls_obs_kf"], -1).astype(np.int32)
    q["ls_obs_le"] = np.concatenate([p["ls_obs_le"], [[1.0, 0.0, -CAM["cx"]]]])
    return q, len(p["pt"]) + len(p["ls"])


def orphan_map(kind):
    p = synth.local_map_problem(CAM, n_kf=3, n_fixed=2, seed=1)
    q = _copy(p)
    q[kind] = np.concatenate([p[kind], p[kind][:1]])   # a landmark without observations
    return q, len(p["pt"]) if kind == "pt" else len(p["pt"]) + len(p["ls"])


# the host loop's exits and its "error grew" branch: (name, map kwargs, opts kwargs, what the trace must show)
BRANCH_MAP = dict(n_kf=5, n_fixed=2, seed=1)
BRANCHES = [
    ("max_iters", {}, dict(max_iters=2), "maxit"),
    ("min_error", {}, dict(min_error=1e3), "min_error"),
    ("min_error_change", {}, {}, "change"),
    ("step", {}, dict(lambda_=1e-3, min_error_change=0.3), "step"),
    ("grew", dict(px_noise=3.0), {}, "grew"),
]


def branch_case(name, quirks):
    _, mkw, okw, _ = [b for b in BRANCHES if b[0] == name][0]
    return synth.local_map_problem(CAM, **dict(BRANCH_MAP, **mkw)), dict(okw, ref_quirks=quirks)


def took(trace, what):
    """whether the oracle's trace shows the branch"""
    last = int(trace["stop"][-1])
    return {"maxit": last == clib.LBA_STOP_MAXIT, "min_error": last == clib.LBA_STOP_MIN_ERROR,
            "change": last == clib.LBA_STOP_CHANGE, "step": last == clib.LBA_STOP_STEP,
            "grew": bool(np.any((trace["applied"][1:] == 0) & (trace["step"][1:] >= 0)))}[what]


def decidable(trace, o, rel=1e-9, step_rel=1e-6):
    """True when every decision the oracle's run took (trace) lies outside the band another summation order can move it
    by: the change test, the error test and `err > err_prev` (only reached when the change test fails) at rel of the
    errors, the |dx| test at step_rel of min_error_change (|dx| comes out of a different solver on the device).  The
    first pass's error is +inf under (q1)."""
    for i in range(1, len(trace)):
        e, ep = float(trace["err"][i]), float(trace["err"][i - 1])
        band = rel * max(abs(e), abs(ep) if np.isfinite(ep) else 0.0)
        if np.isfinite(ep) and abs(abs(e - ep) - o["min_error_change"]) <= band:
            return False
        if np.isfinite(ep) and abs(e - ep) >= o["min_error_change"] and abs(e - ep) <= band:
            return False
        if abs(e - o["min_error"]) <= band:
            return False
        s = float(trace["step"][i])
        if s >= 0 and abs(s - o["min_error_change"]) <= step_rel * o["min_error_change"]:
            return False
    return True


def opts(**kw):
    return clib.lba_opts(**kw)


# ---- tests ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [dict(n_kf=1, n_fixed=2), dict(n_kf=9, n_fixed=3), dict(n_kf=9, n_fixed=0),
                                dict(n_kf=43, n_fixed=2, pts_per_kf=3, ls_per_kf=1, t0=5),
                                dict(n_kf=64, n_fixed=4, pts_per_kf=3, ls_per_kf=1), dict(n_kf=2, n_fixed=0, ls_per_kf=0)])
def test_local_map_generator_shape(kw):
    p = synth.local_map_problem(CAM, seed=3, **kw)
    q = synth.local_map_problem(CAM, seed=3, **kw)
    for k in p:
        if k != "truth":
            assert np.array_equal(p[k], q[k]), k
    n_kf, n_fixed = kw["n_kf"], kw["n_fixed"]
    assert p["kf_pose"].shape == (n_kf, 6) and p["fixed_T"].shape == (n_fixed, 4, 4)
    n_obs, seen_local, seen_fixed = [], [], []
    for kind in ("pt", "ls"):
        lm, kf = p[kind + "_obs_lm"], p[kind + "_obs_kf"]
        assert np.all(np.diff(lm) >= 0)                                   # grouped, ascending
        assert kf.min(initial=0) >= -n_fixed and kf.max(initial=-1) < n_kf
        n = len(p[kind])
        n_obs.append(np.bincount(lm, minlength=n))
        seen_local.append(np.bincount(lm[kf >= 0], minlength=n) > 0)
        seen_fixed.append(np.bincount(lm[kf < 0], minlength=n) > 0)
    n_obs, seen_local, seen_fixed = map(np.concatenate, (n_obs, seen_local, seen_fixed))
    assert n_obs.min() >= 1                                                  # every landmark observed
    assert 0.2 <= np.mean(n_obs == 1) <= 0.4                                 # 20-40 % seen once
    assert np.any(n_obs > 1)
    assert np.any((n_obs == 1) & seen_local)                                 # single observations by local keyframes
    if n_fixed:
        assert np.any(seen_local & ~seen_fixed) and np.any(seen_fixed & ~seen_local) and np.any(seen_fixed & seen_local)
    else:
        assert seen_local.all()
    ident = [np.array_equal(T, np.eye(4)) for T in p["fixed_T"]]
    assert ident == [kw.get("t0", 0) == 0 and i == 0 for i in range(n_fixed)]   # keyframe 0 among the fixed ones or not
    # observations are the projections of the truth plus noise
    T = p["truth"]["T"]
    for j in range(min(20, len(p["pt_obs_kf"]))):
        t = p["pt_obs_kf"][j] + n_fixed if p["pt_obs_kf"][j] >= 0 else -1 - p["pt_obs_kf"][j]
        assert np.abs(_proj(T[t], p["truth"]["pt"][p["pt_obs_lm"][j]]) - p["pt_obs_xy"][j]).max() < 2.0


@pytest.mark.parametrize("homog_th", [1e-7, 1e-3])
def test_edge_maps_put_rows_on_the_edges(homog_th):
    p = edge_map(homog_th)
    n = len(p["pt"]) - 3
    T0inv = np.linalg.inv(synth.expmap_se3(p["kf_pose"][0]))
    depth = lambda P: (T0inv[:3, :3] @ P + T0inv[:3, 3])[2]
    assert 0 < depth(p["pt"][n + 1]) < np.sqrt(homog_th) and 0 < depth(p["ls"][0, :3]) < np.sqrt(homog_th)
    assert depth(p["pt"][n + 2]) < 0
    rows = lambda lm: np.flatnonzero(p["pt_obs_lm"] == lm)
    assert {int(p["pt_obs_kf"][k]) for k in rows(n + 1)} >= {0} and {int(p["pt_obs_kf"][k]) for k in rows(n + 2)} >= {0}
    # the zero residuals are exact in double arithmetic: on an optical axis of the identity
    assert p["pt"][n][0] == 0 and p["pt"][n][1] == 0 and list(p["pt_obs_xy"][rows(n)[0]]) == [CAM["cx"], CAM["cy"]]
    assert p["ls"][1][0] == 0 and p["ls"][1][3] == 0 and p["ls_obs_le"][3].tolist() == [1.0, 0.0, -CAM["cx"]]
    for lm in (n, n + 1, n + 2):
        assert len(rows(lm)) == 3                                                # with well-posed rows
    for quirks in (1, 0):
        r = clib.local_ba(CAM, p, opts(ref_quirks=quirks, homog_th=homog_th))
        assert r["rc"] == 0 and np.isfinite(r["kf_pose"]).all() and np.isfinite(r["pt"]).all() and np.isfinite(r["ls"]).all()
        assert len(r["trace"]) >= 2 and r["trace"]["step"][0] > 1e-3         # the edges do not freeze the map
        assert decidable(r["trace"], opts(ref_quirks=quirks, homog_th=homog_th))


@pytest.mark.parametrize("quirks", [1, 0])
@pytest.mark.parametrize("name", [b[0] for b in BRANCHES])
def test_branch_cases_take_their_branch(name, quirks):
    p, okw = branch_case(name, quirks)
    o = opts(**okw)
    r = clib.local_ba(CAM, p, o)
    tr = r["trace"]
    assert r["rc"] == 0 and took(tr, [b for b in BRANCHES if b[0] == name][0][3]), tr
    assert decidable(tr, o)
    # the trace and the result agree: one record per pass, the counter, the lambda schedule
    maxit = tr["stop"][-1] == clib.LBA_STOP_MAXIT
    assert len(tr) == r["iters"] + (0 if maxit else 1)
    assert np.all(tr["stop"][:-1] == clib.LBA_CONTINUE) and tr["applied"][0] == 1
    lam = tr["lambda_"][0]
    for rec in tr[1:]:
        assert rec["lambda_"] == pytest.approx(lam, rel=1e-12)
        if rec["step"] >= 0:
            lam = lam * 10.0 if rec["applied"] else lam / 10.0
    assert r["lambda_"] == pytest.approx(lam, rel=1e-12)
    assert r["err"] == tr["err"][-1] or (np.isnan(r["err"]) and np.isnan(tr["err"][-1]))


@pytest.mark.parametrize("quirks", [1, 0])
def test_oracle_refuses_landmarks_without_information(quirks):
    for q, lm in (zero_block_map("pt"), zero_block_map("ls"), orphan_map("pt"), orphan_map("ls")):
        r = clib.local_ba(CAM, q, opts(ref_quirks=quirks))
        assert r["rc"] == clib.LBA_ZERO_BLOCK and r["zero_lm"] == lm
        for k in ("kf_pose", "pt", "ls"):
            assert np.array_equal(r[k], np.asarray(q[k]).reshape(r[k].shape)), k   # refused before any step
        g = gba.global_ba(CAM, q, gba.opts(ref_quirks=quirks))
        assert g["rc"] == clib.LBA_ZERO_BLOCK and g["zero_lm"] == lm
    # the same maps without that landmark, and the edge maps, whose zero rows sit beside well-posed ones, are solved
    base = synth.local_map_problem(CAM, n_kf=3, n_fixed=2, seed=1)
    assert clib.local_ba(CAM, base, opts(ref_quirks=quirks))["rc"] == 0
    assert clib.local_ba(CAM, edge_map(1e-7), opts(ref_quirks=quirks))["rc"] == 0


def first_step_residual(p, got, homog_th=1e-7, exact=False):
    """|H DX - g| / |g| for the step recovered from a max_iters = 1 result: H, g the first pass's normal equations
    (oracle/gba.py's rows without GBA's quirks are LBA's first pass), damped by 1e-5 max |H_ii|.  The keyframe part of
    DX is recovered through logmap_se3 of the output pose, which carries about 1e-11 of rounding at these 50 m
    translations: about 1e-9 of residual.  exact: also max |DX - H^-1 g| / max |H^-1 g| (scipy's sparse LU)."""
    import scipy.sparse as sp
    nkf = len(p["kf_pose"])
    X0 = np.concatenate([p["kf_pose"].ravel(), p["pt"].ravel(), p["ls"].ravel()])
    T0inv = np.stack([gba._pose_inv(x) for x in p["kf_pose"]])
    Hl, g, _ = gba.normal_equations(CAM, p, X0, T0inv, True, False, homog_th)
    dg = Hl.diagonal()
    lam = 1e-5 * np.abs(dg).max()
    Hl = Hl + sp.diags(lam * dg)
    H = (Hl + Hl.T - sp.diags(Hl.diagonal())).tocsr()
    # T_out = T_in inverse(exp(dx)): dx = log(T_out^-1 T_in); landmarks: X_out - X_in
    dk = np.stack([clib.logmap_se3(clib.inverse_se3(clib.expmap_se3(a)) @ clib.expmap_se3(b))
                   for a, b in zip(got["kf_pose"], p["kf_pose"])])
    DX = np.concatenate([dk.ravel(), np.concatenate([got["pt"].ravel(), got["ls"].ravel()]) - X0[6 * nkf:]])
    res = np.linalg.norm(H @ DX - g) / np.linalg.norm(g)
    if not exact:
        return res, lam
    import scipy.sparse.linalg as spla
    want = spla.splu(H.tocsc()).solve(g)
    return res, lam, np.abs(DX - want).max() / np.abs(want).max()


BACKWARD_MAPS = {43: dict(n_kf=43, n_fixed=2, pts_per_kf=3, ls_per_kf=1, seed=43),
                 64: dict(n_kf=64, n_fixed=4, pts_per_kf=3, ls_per_kf=1, seed=64)}


@pytest.mark.parametrize("quirks", [1, 0])
def test_oracle_first_step_solves_its_damped_system(quirks):
    p = synth.local_map_problem(CAM, **BACKWARD_MAPS[64])
    r = clib.local_ba(CAM, p, opts(ref_quirks=quirks, max_iters=1))
    assert r["rc"] == 0 and r["iters"] == 1
    res, lam, fwd = first_step_residual(p, r, exact=True)
    assert r["lambda_"] == pytest.approx(lam, rel=1e-12)
    assert fwd <= 1e-10, fwd      # the dense LDL^T's step is scipy's to 1e-10 of the step
    assert res <= 1e-9, res       # ten times the device's bound; the rest is the pose recovery's rounding
