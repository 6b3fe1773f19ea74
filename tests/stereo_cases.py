"""Seeded stereo sequences built to sit on the stereo-association and frame-to-frame gates of the batched pipeline.

Every case derives its right images from its left ones, so the geometry of each correspondence is known exactly: a
textured canvas (synth.scene_pair's left view, or a lattice of tests/adversarial_images.py) is cropped at (x0, y0) for the
left image and at (x0 + dx, y0 + dy) for the right one, so that a level-0 ORB corner at (x, y) on the left sits at
(x - dx, y - dy) on the right: |yl - yr| = dy and d = dx exactly, and the higher octaves land near those values on both
sides.  Frame i of a sequence moves the crop `step` pixels along x (a fronto-parallel scene under a sideways camera).

    shift        dy = 1: the level-0 epipolar differences sit exactly on max_dist_epip = 1
    shift90      dy = 90: some higher-octave differences |yl - yr| round down in f32 (the exact difference is larger)
    shear        row y of the right image shifted by dx + y // shear_div: disparity grows down the image and line
                 disparity ratios span ls_min_disp_ratio
    band         rows of the right image blanked: partly occluded lines take the partial / containing / disjoint
                 overlap branches
    same         L == R: zero disparity everywhere (points at infinity where min_disp <= 0)
    mirror       dx < 0: negative disparities
    lattice      a dot lattice: many equal descriptors, ties in the mutual check
    dense        > 1024 stereo rows of each kind in one pair (several 1024-row chunks of k_stereo_* and k_f2f_build)
    grid1024 / grid1242
                 widths where 64 / width is dyadic and where it is not; shifted by whole grid cells, so that the right
                 features sit on the edges of the (matching_s_ws, 0) x (0, 0) window

build(name) returns dict(cam, frames=[(left, right, None)], prm (plf_params overrides), limits (plf_limits overrides)).
"""
import numpy as np

import adversarial_images as adv
from oracle import frontend as ofe
from oracle import synth

CAM = dict(width=640, height=360, fx=500.0, fy=500.0, cx=320.0, cy=180.0, b=0.537165719)
PAD = 96


def canvas(w, h, seed, **kw):
    """A textured image PAD pixels larger than (w, h) each way (synth.scene_pair's left view, its own noise baked in)."""
    return synth.scene_pair(w=w + 2 * PAD, h=h + 2 * PAD, seed=seed, disparity=0, **kw)[0]


def crop(c, x0, y0, w, h):
    return np.ascontiguousarray(c[y0:y0 + h, x0:x0 + w])


def pair(c, x0, y0, w, h, dx=0, dy=0, shear_div=0, band=None):
    """Left = c at (x0, y0); right = c at (x0 + dx (+ y // shear_div on row y), y0 + dy); band = (r0, r1): right rows r0..r1-1
    set to the background grey."""
    left = crop(c, x0, y0, w, h)
    if shear_div:
        right = np.stack([c[y0 + dy + y, x0 + dx + y // shear_div:x0 + dx + y // shear_div + w] for y in range(h)])
    else:
        right = crop(c, x0 + dx, y0 + dy, w, h)
    right = np.ascontiguousarray(right)
    if band is not None:
        right[band[0]:band[1]] = 90
    return left, right


def sequence(c, w, h, n=3, step=3, **kw):
    return [pair(c, PAD + i * step, PAD, w, h, **kw) + (None,) for i in range(n)]


def lattice_canvas(w, h):
    img, _ = adv.dot_lattice(7, 7, (3, 5), w=w + 2 * PAD, h=h + 2 * PAD, fg=200, bg=60)
    # a few textured rectangles break the lattice's translation symmetry, so that frames still have distinct rows
    tex = canvas(w, h, seed=77, n_rect=40, n_lines=0)
    mask = (np.indices(img.shape).sum(0) // 97) % 5 == 0
    return np.where(mask, tex, img).astype(np.uint8)


def build(name):
    w, h = CAM["width"], CAM["height"]
    prm, lim, cam = {}, {}, CAM
    if name == "shift":
        frames = sequence(canvas(w, h, 11), w, h, dx=12, dy=1)
    elif name == "shift90":
        frames = sequence(canvas(w, h, 11), w, h, dx=12, dy=90)
    elif name == "shear":
        frames = sequence(canvas(w, h, 12), w, h, dx=4, shear_div=12)
    elif name == "band":
        frames = sequence(canvas(w, h, 13, n_lines=260), w, h, dx=10, band=(150, 190))
    elif name == "same":
        frames = sequence(canvas(w, h, 14), w, h, dx=0)
    elif name == "mirror":
        frames = sequence(canvas(w, h, 15), w, h, dx=-8)
    elif name == "lattice":
        frames = sequence(lattice_canvas(w, h), w, h, dx=7)
    elif name == "dense":
        cam = dict(CAM, width=1024, height=512, cx=512.0, cy=256.0)
        w, h = cam["width"], cam["height"]
        frames = sequence(canvas(w, h, 16, n_rect=600, n_lines=400), w, h, n=2, dx=9)
        prm = dict(orb_nfeatures=2000, lsd_nfeatures=0, min_line_length=0.0)
        lim = dict(max_keypoints=4096, max_lines=4096, max_segments=16384)
    elif name in ("grid1024", "grid1242"):
        w = int(name[4:])
        h = 384 if w == 1024 else 375
        cam = dict(CAM, width=w, height=h, cx=w / 2, cy=h / 2)
        cell = w / 64.0
        frames = sequence(canvas(w, h, 17), w, h, dx=int(round(2 * cell)), step=int(round(cell)))
        prm = dict(orb_nfeatures=1500, matching_s_ws=2)
    else:
        raise KeyError(name)
    return dict(cam=cam, frames=frames, prm=prm, limits=lim)


NAMES = ["shift", "shift90", "shear", "band", "same", "mirror", "lattice", "dense", "grid1024", "grid1242"]


# ---- the gates' values on a case's first pair, and parameter settings pinned to a real candidate ---------------------
_DET = {}


def detections(name, k=0):
    """ORB key points / descriptors and LSD KeyLines / LBD descriptors of both images of pair k (oracle, cached)."""
    key = (name, k)
    if key not in _DET:
        c = build(name)
        prm = dict(ofe.DEFAULTS, **c["prm"])
        L, R, _ = c["frames"][k]
        lines = lambda im: ofe.detect_lines(im, prm["lsd_nfeatures"], prm["min_line_length"], ofe.lsd_kwargs(prm))
        _DET[key] = (c, ofe._orb_c(L, prm), ofe._orb_c(R, prm), lines(L), lines(R))
    return _DET[key]


def gate_trace(name, k=0, **over):
    """(points trace, lines trace) of ofe.stereo_points / stereo_lines on pair k of case `name` with `over` applied."""
    c, (kp_l, d_l), (kp_r, d_r), (kl_l, ld_l), (kl_r, ld_r) = detections(name, k)
    prm = dict(ofe.DEFAULTS, **c["prm"], **over)
    _, tp = ofe.stereo_points(c["cam"], kp_l, d_l, kp_r, d_r, prm, trace=True)
    _, tl = ofe.stereo_lines(c["cam"], kl_l, ld_l, kl_r, ld_r, prm, trace=True)
    return tp, tl


def below(v):
    return float(np.nextafter(np.float32(v), np.float32(-np.inf)))


def above(v):
    return float(np.nextafter(np.float32(v), np.float32(np.inf)))


def bracket(x):
    """The two floats around the double x: (largest float <= x, the next one up)."""
    lo = np.float32(x)
    if float(lo) > x:
        lo = np.nextafter(lo, np.float32(-np.inf))
    return float(lo), above(lo)


def _flips(name, kind, row, param, accept, reject, strategy):
    """Candidate `row` (left index) of pair 0 is accepted at param = accept and rejected at param = reject."""
    got = []
    for v in (accept, reject):
        t = gate_trace(name, matching_strategy=strategy, **{param: v})[0 if kind == "pt" else 1]
        sel = t["ok"][t["i"] == row]
        got.append(bool(sel[0]) if len(sel) else None)
    return got == [True, False]


def _pick(name, kind, param, cands, settings, strategy):
    """The first candidate (trace row index list `cands`) whose decision flips between the two settings."""
    for r in cands:
        acc, rej = settings(r)
        if _flips(name, kind, r["i"], param, acc, rej, strategy):
            return r, float(acc), float(rej)
    raise AssertionError(f"no candidate of {name} flips {param} at matching_strategy {strategy}")


def _rows(t, mask):
    return [{k: v[n] for k, v in t.items()} for n in np.nonzero(mask)[0]]


# the pins of each matching strategy.  epip_f32 needs |yl - yr| far above a grid cell's height: the windowed stereo
# match ((matching_s_ws, 0) x (0, 0) cells) only pairs key points of one cell row, whose f32 differences are exact
PIN_LABELS = {0: ["epip", "epip_f32", "min_disp_pt", "horiz", "overlap_one", "overlap", "ratio", "min_disp_ls"],
              3: ["epip", "min_disp_pt", "horiz", "overlap_one", "overlap", "ratio", "min_disp_ls"]}


def pins(strategy=0):
    """[(label, case, parameter, accepting value, rejecting value, candidate's trace row)] at matching_strategy
    `strategy`: each setting pair is the f32 value a real candidate of the case's first pair produces (or the floats
    bracketing a double one) and its neighbour, so that the candidate's own gate alone decides it."""
    out = []
    tr = lambda name, **over: gate_trace(name, matching_strategy=strategy, **over)
    pick = lambda name, kind, param, cands, settings: _pick(name, kind, param, cands, settings, strategy)
    # epipolar gate: a level-0 correspondence of the dy = 1 shift sits exactly on max_dist_epip = 1 (<= accepts it)
    tp, _ = tr("shift", max_dist_epip=1e9)
    m = (tp["d"] >= 1.0) & (tp["epip"] == 1.0)
    r, a, b = pick("shift", "pt", "max_dist_epip", _rows(tp, m), lambda r: (r["epip"], below(r["epip"])))
    out.append(("epip", "shift", "max_dist_epip", a, b, r))
    if "epip_f32" in PIN_LABELS[strategy]:
        # a difference that f32 rounds down (yl, yr 90 rows apart): max_dist_epip = its f32 value accepts it, and the
        # exact (double) difference would not
        tp, _ = tr("shift90", max_dist_epip=1e9)
        m = (tp["d"] >= 1.0) & (tp["epip"] < tp["epip_f64"])
        r, a, b = pick("shift90", "pt", "max_dist_epip", _rows(tp, m), lambda r: (r["epip"], below(r["epip"])))
        out.append(("epip_f32", "shift90", "max_dist_epip", a, b, r))
    # point disparity: d itself (>= accepts it)
    tp, _ = tr("shift")
    m = tp["epip_ok"] & (tp["d"] > 1.0)
    r, a, b = pick("shift", "pt", "min_disp", _rows(tp, m), lambda r: (r["d"], above(r["d"])))
    out.append(("min_disp_pt", "shift", "min_disp", a, b, r))
    # line horizontality: a right line whose |r0| rounds down to f32, so that the f32 value is rejected and the double
    # is not
    _, tl = tr("band")
    m = tl["ratio_ok"] & tl["disp_ok"] & tl["overlap_ok"] & (np.abs(tl["r0"]) > tl["horiz"])
    r, a, b = pick("band", "ls", "line_horiz_th", _rows(tl, m), lambda r: (below(r["horiz"]), r["horiz"]))
    out.append(("horiz", "band", "line_horiz_th", a, b, r))
    # overlap: exactly 1 (a float: > rejects it) and a double one between two floats
    m = tl["ratio_ok"] & tl["disp_ok"] & tl["horiz_ok"] & (tl["overlap"] == 1.0)
    r, a, b = pick("band", "ls", "stereo_overlap_th", _rows(tl, m), lambda r: (below(1.0), 1.0))
    out.append(("overlap_one", "band", "stereo_overlap_th", a, b, r))
    m = tl["ratio_ok"] & tl["disp_ok"] & tl["horiz_ok"] & (tl["overlap"] > 0.8) & (tl["overlap"] < 1.0)
    r, a, b = pick("band", "ls", "stereo_overlap_th", _rows(tl, m), lambda r: bracket(r["overlap"]))
    out.append(("overlap", "band", "stereo_overlap_th", a, b, r))
    # disparity ratio of a sheared line
    _, tl = tr("shear", ls_min_disp_ratio=0.0)
    m = tl["ok"] & (tl["ratio"] > 0.6) & (tl["ratio"] < 0.95)
    r, a, b = pick("shear", "ls", "ls_min_disp_ratio", _rows(tl, m), lambda r: bracket(r["ratio"]))
    out.append(("ratio", "shear", "ls_min_disp_ratio", a, b, r))
    # line disparity: the smaller end's disparity, bracketed
    _, tl = tr("shear")
    m = tl["ok"]
    r, a, b = pick("shear", "ls", "min_disp", _rows(tl, m), lambda r: bracket(min(r["disp_s"], r["disp_e"])))
    out.append(("min_disp_ls", "shear", "min_disp", a, b, r))
    return out


def fallback_pins(name="shear"):
    """The match() fall-back of the windowed tracking (k_mg_select), on case `name`'s first two pairs ordered so that the
    previous frame holds more stereo rows of each kind than the current one, at matching_strategy 3: for points and lines,
    [(label, frames, overrides)] with min_*_matches = the oracle's windowed count n (no fall-back), n + 1 (fall-back) and
    the current frame's row count (both frames must hold more than that: no fall-back)."""
    c = build(name)
    prm = dict(ofe.DEFAULTS, **c["prm"], matching_strategy=3)
    frames = c["frames"][:2]
    f = [ofe.extract_stereo(c["cam"], L, R, prm) for L, R, _ in frames]
    if len(f[0].pdesc) < len(f[1].pdesc):
        frames, f = frames[::-1], f[::-1]
    prev, curr = f
    w = (int(prm["matching_f2f_ws"]),) * 4
    _, n_pt = ofe.grid_match_points(c["cam"], ofe.projection(c["cam"], prev.pt_P), prev.pdesc, curr.pt_pl, curr.pdesc, w,
                                    prm["min_ratio_12_p"], prm["best_lr_matches"])
    q = np.concatenate([ofe.projection(c["cam"], prev.ls_sP), ofe.projection(c["cam"], prev.ls_eP)], 1)
    _, n_ls = ofe.grid_match_lines(c["cam"], q, prev.ldesc, np.concatenate([curr.ls_spl, curr.ls_epl], 1), curr.ldesc, w,
                                   prm["min_ratio_12_l"], prm["line_sim_th"], prm["best_lr_matches"])
    counts = dict(pt=(len(prev.pdesc), len(curr.pdesc), int(n_pt)), ls=(len(prev.ldesc), len(curr.ldesc), int(n_ls)))
    out = []
    for kind, key in (("pt", "min_pt_matches"), ("ls", "min_ls_matches")):
        _, n_curr, n = counts[kind]
        for label, v in (("n", n), ("n+1", n + 1), ("n_curr", n_curr)):
            out.append((f"{kind}_{label}", frames, {key: v}))
    return out, counts
