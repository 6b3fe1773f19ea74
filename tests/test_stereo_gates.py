"""CPU checks of tests/stereo_cases.py: the oracle's gate trace agrees with what stereo_points / stereo_lines return, and
every case reaches what it is built for, measured with numbers - each pinned candidate flips between neighbouring
settings, every overlap branch is taken, more than 1024 stereo and tracked rows of each kind occur in one pair, tied
descriptors occur, key points sit on grid-cell boundaries and the previous frame projects to NaN where L == R.
tests/test_stereo_gates_gpu.py runs the same cases and settings through the batched pipeline."""
import numpy as np
import pytest

import stereo_cases as sc
from oracle import frontend as ofe
from oracle import matching as om


@pytest.mark.parametrize("name", sc.NAMES)
def test_trace_agrees_with_outputs(built, name):
    c, (kp_l, d_l), (kp_r, d_r), (kl_l, ld_l), (kl_r, ld_r) = sc.detections(name)
    for strategy in (0, 3):
        prm = dict(ofe.DEFAULTS, **c["prm"], matching_strategy=strategy)
        pts, tp = ofe.stereo_points(c["cam"], kp_l, d_l, kp_r, d_r, prm, trace=True)
        assert np.array_equal(pts[0], ofe.stereo_points(c["cam"], kp_l, d_l, kp_r, d_r, prm)[0])
        ok = tp["i"][tp["ok"]]
        assert np.array_equal(pts[4], d_l[ok]) and np.array_equal(pts[0][:, 0], kp_l["x"][ok].astype(np.float64))
        assert np.array_equal(pts[1], tp["d"][tp["ok"]])
        assert np.array_equal(tp["ok"], tp["epip_ok"] & tp["disp_ok"])
        ls, tl = ofe.stereo_lines(c["cam"], kl_l, ld_l, kl_r, ld_r, prm, trace=True)
        ok = tl["i"][tl["ok"]]
        assert np.array_equal(ls[8], ld_l[ok]) and np.array_equal(ls[0][:, 0], kl_l["startPointX"][ok].astype(np.float64))
        assert np.array_equal(tl["ok"], tl["disp_ok"] & tl["horiz_ok"] & tl["overlap_ok"])
        assert np.array_equal(ls[2], tl["disp_s"][tl["ok"]]) and np.array_equal(ls[3], tl["disp_e"][tl["ok"]])
        assert not (tl["disp_ok"] & ~tl["ratio_ok"]).any()


@pytest.mark.parametrize("strategy", [0, 3])
def test_pinned_candidates_flip(built, strategy):
    """Each pinned setting pair accepts its candidate at one value and rejects it at the neighbouring float, at the
    matching strategy it is pinned for (the candidate is paired by that strategy's stereo match)."""
    pins = sc.pins(strategy)
    assert [p[0] for p in pins] == sc.PIN_LABELS[strategy]
    for label, name, param, acc, rej, row in pins:
        assert np.float32(acc) == acc and np.float32(rej) == rej, label               # C floats
        assert abs(np.nextafter(np.float32(acc), np.float32(rej)) - np.float32(rej)) == 0, label   # neighbours
        kind = 1 if param in ("line_horiz_th", "stereo_overlap_th", "ls_min_disp_ratio") or label == "min_disp_ls" else 0
        for v, want in ((acc, True), (rej, False)):
            t = sc.gate_trace(name, matching_strategy=strategy, **{param: v})[kind]
            assert bool(t["ok"][t["i"] == row["i"]][0]) is want, (label, v)
        print(f"strategy {strategy} {label}: {param} {acc!r} accepts, {rej!r} rejects left row {row['i']} of {name}")
    by = {p[0]: p for p in pins}
    assert by["epip"][3] == 1.0 == ofe.DEFAULTS["max_dist_epip"]     # the default gate sits on the dy = 1 correspondences
    assert by["overlap_one"][4] == 1.0
    h = by["horiz"][5]
    assert abs(h["r0"]) > h["horiz"] == by["horiz"][4]                 # f32 |r0| is rejected where the double would pass
    if strategy == 0:
        e = by["epip_f32"][5]
        assert e["epip"] == by["epip_f32"][3] < e["epip_f64"]          # f32 accepts at its own value, the double would not
    else:
        # one cell row of the windowed stereo match: no f32 epipolar difference rounds, in any case
        for name in sc.NAMES:
            tp, _ = sc.gate_trace(name, matching_strategy=3, max_dist_epip=1e9)
            assert not (tp["epip"] < tp["epip_f64"]).any(), name


def test_fallback_settings_straddle_the_decision(built):
    pins, counts = sc.fallback_pins()
    for kind in ("pt", "ls"):
        n_prev, n_curr, n = counts[kind]
        assert n_prev > n_curr > n > 0, (kind, counts)                  # at kmin = n_curr only n2 > kmin decides
    labels = [p[0] for p in pins]
    assert labels == ["pt_n", "pt_n+1", "pt_n_curr", "ls_n", "ls_n+1", "ls_n_curr"]


def test_every_overlap_branch_is_taken(built):
    seen, clamped = {}, 0
    for name in sc.NAMES:
        for strategy in (0, 3):
            _, tl = sc.gate_trace(name, matching_strategy=strategy)
            for b in ("horizontal", "disjoint", "containing", "partial"):
                seen[b] = seen.get(b, 0) + int((tl["branch"] == b).sum())
            seen["short"] = seen.get("short", 0) + int(tl["short"].sum())
            clamped += int(tl["clamped"].sum())
    print("overlap branches over the cases:", seen, "clamped:", clamped)
    assert all(v > 0 for v in seen.values()), seen
    # the > 1 clamp cannot act: length = eln - spn bounds both the containing (eln - sln, sln > spn) and the partial
    # (min(eln, epn) - max(sln, spn)) overlaps, so overlap / length <= 1 whenever length > 0.01
    assert clamped == 0


def test_more_than_1024_rows_in_one_pair(built):
    c = sc.build("dense")
    prm = dict(ofe.DEFAULTS, **c["prm"])
    f = [ofe.extract_stereo(c["cam"], L, R, prm) for L, R, _ in c["frames"]]
    tr = ofe.track(f[0], f[1], prm, cam=c["cam"])
    n = dict(pt=len(f[0].pt_pl), ls=len(f[0].ls_spl), pt_tracked=len(tr["P"]), ls_tracked=len(tr["sP"]))
    print("dense pair:", n)
    assert min(n.values()) > 1024, n
    # the rows of the last 1024-row chunk are accepted too (a lost chunk offset would overwrite earlier rows)
    tp, tl = sc.gate_trace("dense")
    assert (tp["ok"] & (tp["i"] >= 1024)).any() and (tl["ok"] & (tl["i"] >= 1024)).any()


def test_lattice_has_tied_descriptors(built):
    c, (kp_l, d_l), (kp_r, d_r), _, _ = sc.detections("lattice")
    dist = om.hamming_matrix(d_l, d_r)
    s = np.sort(dist, 1)
    ties = int((s[:, 0] == s[:, 1]).sum())
    dup = len(d_l) - len(np.unique(d_l, axis=0))
    print(f"lattice: {ties} left key points with two equal best distances, {dup} repeated descriptors")
    assert ties > 100 and dup > 0


@pytest.mark.parametrize("name", ["grid1024", "grid1242"])
def test_key_points_on_cell_boundaries(built, name):
    c, (kp_l, _), (kp_r, _), _, _ = sc.detections(name)
    iw, ih = ofe.grid_scales(c["cam"])
    on = 0
    for kp in (kp_l, kp_r):
        sx, sy = kp["x"].astype(np.float64) * iw, kp["y"].astype(np.float64) * ih
        on += int(((sx == np.trunc(sx)) | (sy == np.trunc(sy))).sum())
    print(f"{name}: {on} key points on a cell boundary")
    assert on >= (100 if name == "grid1024" else 3)   # 64 / 1242 is not dyadic: few pixel positions scale to an integer


def test_points_at_infinity_project_to_nan(built):
    c = sc.build("same")
    prm = dict(ofe.DEFAULTS, **c["prm"], min_disp=0.0)
    f = ofe.extract_stereo(c["cam"], *c["frames"][0][:2], prm)
    assert len(f.pt_P) > 500 and np.isinf(f.pt_P[:, 2]).all() and (f.pt_disp == 0).all()
    with np.errstate(invalid="ignore", divide="ignore"):
        q = ofe.projection(c["cam"], f.pt_P)
    assert np.isnan(q).all()
    iw, ih = ofe.grid_scales(c["cam"])
    assert (ofe._cell(q[:, 0] * iw) == 0).all() and (ofe._cell(q[:, 1] * ih) == 0).all()   # NaN -> cell 0
    assert ofe._cell(np.array([np.inf]))[0] == ofe.CELL_LIM and ofe._cell(np.array([-2.0 ** 40]))[0] == -ofe.CELL_LIM
    assert len(f.ls_spl) == 0      # 0 / 0 disparity ratios: no line survives
    # with the default min_disp nothing at zero disparity is a stereo row
    assert len(ofe.extract_stereo(c["cam"], *c["frames"][0][:2], dict(ofe.DEFAULTS, **c["prm"])).pt_P) == 0


@pytest.mark.parametrize("strategy", [0, 3])
def test_pose_solver_on_rows_at_infinity(built, strategy):
    """What DESIGN.md §8 states for the oracle's pose solver on rows at infinity (L == R, min_disp = 0; the windowed
    path's NaN queries look around cell 0 with matching_f2f_ws = 10): status 0, DT = identity, every point row an
    inlier, NaN error and covariance, one iteration per stage.  test_stereo_gates_gpu.py holds the device to the same."""
    c = sc.build("same")
    prm = dict(ofe.DEFAULTS, **c["prm"], min_disp=0.0, matching_strategy=strategy, matching_f2f_ws=10, min_pt_matches=0,
               min_ls_matches=0)
    for r in ofe.run_sequence(c["cam"], [(a, b) for a, b, _ in c["frames"]], prm)[1:]:
        res = r["res"]
        n = len(res["inlier_pt"])
        assert r["status"] == 0 and n > (500 if strategy == 0 else 20) and len(res["inlier_ls"]) == 0
        assert np.isinf(res["rows"]["P"]).any(axis=1).all()
        assert np.array_equal(r["DT"], np.eye(4)) and res["n_inliers"] == (n, 0)
        assert np.isnan(res["err"]) and np.isnan(res["cov"]).all() and tuple(res["iters"]) == (1, 1)
