"""TEST INFRASTRUCTURE (oracle) - CPU restatement of the matching and gate parts of MapHandler::matchKF2KFPoints /
matchKF2KFLines (src/mapHandler.cpp:234-278, :365-426) and matchMap2KFPoints / matchMap2KFLines (:532-632, :634-752), the
functions lookForCommonMatches calls (:754-821).  The control flow below is the reference's own (in-tree); matchGrid()
(oracle/matchgrid.py) and match() (oracle/matching.py) keep their "parity unpinned" status (stvo-pl is not vendored).

Reproduced as written:
  - a kind returns 0 when disabled or the keyframe has no stereo features of it (:243, :368, :542, :644); KF-to-KF also
    when the previous keyframe has none; map-to-KF also when no landmark is visible or no feature unmatched (:571, :676);
  - projection cam->projection(R X + t), each row ((r0 x + r1 y) + r2 z) + t; cells = int(v * GRID_COLS / width),
    int(v * GRID_ROWS / height);
  - map visibility pf.x > 0 && pf.x < width && pf.y > 0 && pf.y < height && Z > 0 (:551), both end points for lines
    (:654-655); landmarks kept in index order among the used, visible ones; train = unmatched features in order;
  - matchKF2KFLines leaves the projected query lines in PIXELS (:392-393, unlike :256 and :658-659);
  - fallback to match(): KF-to-KF n_curr > min && n_prev > min && matches < min (:274-276, :421-423); map-to-KF tests the
    visible-landmark count twice (:594-595, :709-710); without fast_matching `matches` is 0 and, fallback not taken, there
    are no pairs;
  - map gates on the surviving pairs: |pf_map - pl| < max_kf_epip_p (:612-613); lines le . (p, 1) < max_kf_epip_l at both
    projected end points, SIGNED (:727-729); each reject decrements the return value (:628, :748).
One definition of this library: query cells are clamped to +-2^28 before the double -> int conversion (undefined in the
reference beyond int range) and NaN becomes 0; the Bresenham walk of a query line only visits the steps whose window can
reach the grid (the others add no candidate)."""
import numpy as np

from oracle import matching as om
from oracle import matchgrid as mg
from oracle.frontend import GRID_COLS, GRID_ROWS

CELL_LIM = float(1 << 28)


def rigid(T, X):
    """R X + t with the row order ((r0 x + r1 y) + r2 z) + t (f64, no contraction)."""
    T = np.asarray(T, np.float64).reshape(4, 4)
    X = np.asarray(X, np.float64).reshape(-1, 3)
    x, y, z = X[:, 0], X[:, 1], X[:, 2]
    return np.stack([((T[r, 0] * x + T[r, 1] * y) + T[r, 2] * z) + T[r, 3] for r in range(3)], 1)


def project(cam, P):
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.stack([cam["cx"] + cam["fx"] * P[:, 0] / P[:, 2], cam["cy"] + cam["fy"] * P[:, 1] / P[:, 2]], 1)


def qcell(v):
    v = np.asarray(v, np.float64)
    out = np.trunc(np.clip(v, -CELL_LIM, CELL_LIM))
    return np.where(np.isnan(v), 0, out).astype(np.int64)


def tcell(v):
    return np.trunc(np.asarray(v, np.float64)).astype(np.int64)


def _walk_clipped(x1, y1, x2, y2, w):
    """The cells of bresenham(x1, y1, x2, y2) whose window (w) can reach the grid, in walk order."""
    x1, y1, x2, y2 = int(x1), int(y1), int(x2), int(y2)
    steep = abs(y2 - y1) > abs(x2 - x1)
    if steep:
        x1, y1, x2, y2 = y1, x1, y2, x2
    if x1 > x2:
        x1, x2, y1, y2 = x2, x1, y2, y1
    dx, dy = x2 - x1, abs(y2 - y1)
    e0, ystep = dx // 2, (1 if y1 < y2 else -1)
    lo = -w[3] if steep else -w[1]
    hi = (GRID_ROWS - 1 + w[2]) if steep else (GRID_COLS - 1 + w[0])
    n0, n_end = max(0, lo - x1), min(x2, hi) - x1
    out = []
    if n0 > n_end:
        return out
    err, y = e0, y1
    if n0 > 0:
        err = (e0 - n0 * dy) % dx
        y = y1 + ystep * ((err - e0 + n0 * dy) // dx)
    for n in range(n0, n_end + 1):
        xx = x1 + n
        out.append((y, xx) if steep else (xx, y))
        err -= dy
        if err < 0:
            y += ystep
            err += dx
    return out


def _grid_lines(q_line, d1, t_line, t_dir, d2, w, nnr, line_sim_th, best_lr):
    """matchGrid (lines) with the clipped query walk (same candidates as oracle/matchgrid.py match_grid_lines)."""
    grid = mg.grid_from_lines(t_line, GRID_ROWS, GRID_COLS)
    q_line = np.asarray(q_line, np.int64).reshape(-1, 4)
    n2 = len(d2)

    def cand(i1):
        c = set()
        for (x, y) in _walk_clipped(*q_line[i1], w):
            c |= grid.get(x, y, w)
        vx, vy = float(q_line[i1, 2] - q_line[i1, 0]), float(q_line[i1, 3] - q_line[i1, 1])
        with np.errstate(invalid="ignore", divide="ignore"):
            nrm = np.sqrt(np.float64(vx * vx + vy * vy))
            vx, vy = np.float64(vx) / nrm, np.float64(vy) / nrm
        out = []
        for i2 in sorted(c):
            if not (0 <= i2 < n2):
                continue
            with np.errstate(invalid="ignore"):
                if abs(vx * t_dir[i2, 0] + vy * t_dir[i2, 1]) < line_sim_th:
                    continue
            out.append(i2)
        return out

    return mg._greedy(len(q_line), n2, cand, d1, d2, nnr, best_lr)


def _scales(cam):
    return GRID_COLS / float(cam["width"]), GRID_ROWS / float(cam["height"])


def _train_lines(cam, spl, epl):
    iw, ih = _scales(cam)
    spl, epl = np.asarray(spl, np.float64).reshape(-1, 2), np.asarray(epl, np.float64).reshape(-1, 2)
    t_line = np.stack([tcell(spl[:, 0] * iw), tcell(spl[:, 1] * ih), tcell(epl[:, 0] * iw), tcell(epl[:, 1] * ih)], 1)
    vx, vy = (epl[:, 0] - spl[:, 0]) * iw, (epl[:, 1] - spl[:, 1]) * ih
    with np.errstate(invalid="ignore", divide="ignore"):
        nrm = np.sqrt(vx * vx + vy * vy)
        t_dir = np.stack([vx / nrm, vy / nrm], 1)
    return t_line, t_dir


def _match_kind(prm, fast, lines, q_cells, d1, t_geo, d2, n_cond, kmin):
    """matches_12 and the count after matchGrid (fast) and the match() fallback; n_cond: the fallback's two counts."""
    ws = int(prm["matching_f2f_ws"])
    w = (ws, ws, ws, ws)
    nnr = prm["min_ratio_12_l"] if lines else prm["min_ratio_12_p"]
    best_lr = bool(prm["best_lr_matches"])
    m12, matches = np.full(len(d1), -1, np.int32), 0
    if fast:
        if lines:
            t_line, t_dir = t_geo
            m12, matches = _grid_lines(q_cells, d1, t_line, t_dir, d2, w, nnr, float(np.float32(prm["line_sim_th"])), best_lr)
        else:
            m12, matches = mg.match_grid_points(q_cells, d1, mg.grid_from_points(t_geo, GRID_ROWS, GRID_COLS), d2, w, nnr,
                                                best_lr)
    if n_cond[0] > kmin and n_cond[1] > kmin and matches < kmin:
        m12, matches = om.match(d1, d2, nnr, best_lr)
    return np.asarray(m12, np.int32), int(matches)


def match_kf2kf(cam, prm, prev, curr, DT, fast_matching=True):
    """matchKF2KFPoints + matchKF2KFLines: prev / curr = dicts in get_frame layout.  Returns (m_pt, n_pt, m_ls, n_ls)."""
    iw, ih = _scales(cam)
    n_p, n_c = len(prev["pdesc"]), len(curr["pdesc"])
    m_pt, n_pt = np.full(n_p, -1, np.int32), 0
    if prm.get("has_points", True) and n_p and n_c:                       # :243
        pj = project(cam, rigid(DT, prev["pt_P"]))                         # :255-256 (scaled)
        q = np.stack([qcell(pj[:, 0] * iw), qcell(pj[:, 1] * ih)], 1)
        pl = np.asarray(curr["pt_pl"], np.float64).reshape(-1, 2)
        t = np.stack([tcell(pl[:, 0] * iw), tcell(pl[:, 1] * ih)], 1)     # :260-264
        m_pt, n_pt = _match_kind(prm, fast_matching, False, q, prev["pdesc"], t, curr["pdesc"], (n_c, n_p),
                                 int(prm["min_pt_matches"]))
    n_p, n_c = len(prev["ldesc"]), len(curr["ldesc"])
    m_ls, n_ls = np.full(n_p, -1, np.int32), 0
    if prm.get("has_lines", True) and n_p and n_c:                        # :368
        s, e = project(cam, rigid(DT, prev["ls_sP"])), project(cam, rigid(DT, prev["ls_eP"]))
        q = np.stack([qcell(s[:, 0]), qcell(s[:, 1]), qcell(e[:, 0]), qcell(e[:, 1])], 1)   # :392-393: pixels
        m_ls, n_ls = _match_kind(prm, fast_matching, True, q, prev["ldesc"], _train_lines(cam, curr["ls_spl"], curr["ls_epl"]),
                                 curr["ldesc"], (n_c, n_p), int(prm["min_ls_matches"]))
    return m_pt, n_pt, m_ls, n_ls


def _visible(cam, p, Z):
    return (p[:, 0] > 0) & (p[:, 0] < cam["width"]) & (p[:, 1] > 0) & (p[:, 1] < cam["height"]) & (Z > 0.0)


def match_map2kf(cam, prm, local_map, Twf, kf, kf_pt_lm=None, kf_ls_lm=None, fast_matching=True, max_kf_epip_p=1.0,
                 max_kf_epip_l=1.0):
    """matchMap2KFPoints + matchMap2KFLines.  local_map: dict pt_X [n,3], pt_desc, pt_use (or None), ls_X [n,6], ls_desc,
    ls_use; kf: get_frame dict.  Returns (lm_pt, n_pt, lm_ls, n_ls): per landmark the matched keyframe feature or -1."""
    iw, ih = _scales(cam)
    out = []
    for lines in (False, True):
        key = "ls" if lines else "pt"
        X = np.asarray(local_map[key + "_X"], np.float64).reshape(-1, 6 if lines else 3)
        n_lm = len(X)
        lm_out, n = np.full(n_lm, -1, np.int32), 0
        kdesc = kf["ldesc" if lines else "pdesc"]
        enabled = prm.get("has_lines" if lines else "has_points", True)
        if enabled and len(kdesc) and n_lm:                                 # :542 / :644
            use = local_map.get(key + "_use")
            use = np.ones(n_lm, bool) if use is None else np.asarray(use).astype(bool)
            if lines:
                Ps, Pe = rigid(Twf, X[:, :3]), rigid(Twf, X[:, 3:])
                ps, pe = project(cam, Ps), project(cam, Pe)
                vis = _visible(cam, ps, Ps[:, 2]) & _visible(cam, pe, Pe[:, 2])   # :654-655
            else:
                Pf = rigid(Twf, X)
                ps = project(cam, Pf)
                vis = _visible(cam, ps, Pf[:, 2])                                # :551
            qi = np.nonzero(use & vis)[0]                                        # landmark order
            lm = kf_ls_lm if lines else kf_pt_lm
            ti = np.arange(len(kdesc)) if lm is None else np.nonzero(np.asarray(lm) == -1)[0]   # :565 / :670
            if len(qi) and len(ti):                                              # :571 / :676
                d1 = np.asarray(local_map[key + "_desc"], np.uint8).reshape(-1, 32)[qi]
                d2 = np.asarray(kdesc, np.uint8)[ti]
                if lines:
                    q = np.stack([qcell(ps[qi, 0] * iw), qcell(ps[qi, 1] * ih), qcell(pe[qi, 0] * iw), qcell(pe[qi, 1] * ih)], 1)
                    tg = _train_lines(cam, np.asarray(kf["ls_spl"])[ti], np.asarray(kf["ls_epl"])[ti])
                else:
                    q = np.stack([qcell(ps[qi, 0] * iw), qcell(ps[qi, 1] * ih)], 1)
                    pl = np.asarray(kf["pt_pl"], np.float64)[ti]
                    tg = np.stack([tcell(pl[:, 0] * iw), tcell(pl[:, 1] * ih)], 1)
                kmin = int(prm["min_ls_matches" if lines else "min_pt_matches"])
                m12, n = _match_kind(prm, fast_matching, lines, q, d1, tg, d2, (len(qi), len(qi)), kmin)   # :594-595
                for j, t in enumerate(m12):
                    if t < 0:
                        continue
                    i, f = qi[j], ti[t]
                    if lines:
                        le = np.asarray(kf["ls_le"], np.float64)[f]
                        e0 = le[0] * ps[i, 0] + le[1] * ps[i, 1] + le[2]
                        e1 = le[0] * pe[i, 0] + le[1] * pe[i, 1] + le[2]
                        ok = e0 < max_kf_epip_l and e1 < max_kf_epip_l            # :727-729 (signed)
                    else:
                        pl = np.asarray(kf["pt_pl"], np.float64)[f]
                        dx, dy = ps[i, 0] - pl[0], ps[i, 1] - pl[1]
                        ok = np.sqrt(dx * dx + dy * dy) < max_kf_epip_p          # :612-613
                    if ok:
                        lm_out[i] = f
                    else:
                        n -= 1                                                   # :628 / :748
        out += [lm_out, n]
    return tuple(out)
