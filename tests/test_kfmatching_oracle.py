"""CPU tests of oracle/kfmatching.py: each rule of MapHandler's keyframe / local-map matching it restates
(src/mapHandler.cpp:234-278, :365-426, :532-632, :634-752) on a small hand-built case."""
import numpy as np

from oracle import frontend as ofe
from oracle import kfmatching as kfm

# fx = fy = 512 and Z = 2 make the projections of the hand-built points exact in f64
CAM = dict(width=640, height=480, fx=512.0, fy=512.0, cx=320.0, cy=240.0, b=0.5)
I4 = np.eye(4)


def prm(**kw):
    return dict(ofe.DEFAULTS, **kw)


def descs(n, seed=0):
    return np.random.default_rng(seed).integers(0, 256, (n, 32), dtype=np.uint8)


def back(u, v, Z=2.0):
    """The camera-frame point projecting to pixel (u, v) at depth Z."""
    return np.array([(u - CAM["cx"]) * Z / CAM["fx"], (v - CAM["cy"]) * Z / CAM["fy"], Z])


def points_frame(px, desc, with_P=True):
    px = np.asarray(px, np.float64).reshape(-1, 2)
    f = dict(pt_pl=px, pdesc=desc, ldesc=np.zeros((0, 32), np.uint8))
    if with_P:
        f["pt_P"] = np.array([back(u, v) for u, v in px]).reshape(-1, 3)
    return f


def lines_frame(se, desc):
    se = np.asarray(se, np.float64).reshape(-1, 4)
    le = []
    for sx, sy, ex, ey in se:
        l = np.cross([sx, sy, 1.0], [ex, ey, 1.0])
        le.append(l / np.hypot(l[0], l[1]))
    return dict(pdesc=np.zeros((0, 32), np.uint8), ls_spl=se[:, :2], ls_epl=se[:, 2:],
                ls_sP=np.array([back(*p[:2]) for p in se]).reshape(-1, 3), ls_eP=np.array([back(*p[2:]) for p in se]).reshape(-1, 3),
                ls_le=np.array(le).reshape(-1, 3), ldesc=desc)


def test_early_exits():
    d = descs(12)
    px = np.stack([np.linspace(50, 600, 12), np.linspace(40, 440, 12)], 1)
    f = points_frame(px, d)
    empty = points_frame(np.zeros((0, 2)), d[:0])
    m_pt, n_pt, m_ls, n_ls = kfm.match_kf2kf(CAM, prm(has_points=False), f, f, I4)
    assert n_pt == 0 and (m_pt == -1).all() and len(m_ls) == 0
    m_pt, n_pt, _, _ = kfm.match_kf2kf(CAM, prm(), f, empty, I4)      # current keyframe without points
    assert n_pt == 0 and (m_pt == -1).all()
    m_pt, n_pt, _, _ = kfm.match_kf2kf(CAM, prm(), empty, f, I4)      # previous keyframe without points
    assert n_pt == 0 and len(m_pt) == 0
    m_pt, n_pt, _, _ = kfm.match_kf2kf(CAM, prm(), f, f, I4)
    assert n_pt == 12 and np.array_equal(m_pt, np.arange(12))
    lmap = dict(pt_X=f["pt_P"], pt_desc=d, ls_X=np.zeros((0, 6)), ls_desc=np.zeros((0, 32)))
    lm, n, _, _ = kfm.match_map2kf(CAM, prm(), lmap, I4, f)
    assert n == 12 and np.array_equal(lm, np.arange(12))
    behind = np.diag([1.0, 1.0, -1.0, 1.0])                            # nothing visible
    lm, n, _, _ = kfm.match_map2kf(CAM, prm(), lmap, behind, f)
    assert n == 0 and (lm == -1).all()
    lm, n, _, _ = kfm.match_map2kf(CAM, prm(), lmap, I4, f, kf_pt_lm=np.arange(12))   # every feature matched already
    assert n == 0 and (lm == -1).all()
    lm, n, _, _ = kfm.match_map2kf(CAM, prm(has_points=False), lmap, I4, f)
    assert n == 0 and (lm == -1).all()


def test_strict_visibility_bounds():
    """pf.x > 0 && pf.x < width && pf.y > 0 && pf.y < height && Z > 0 (:551): exactly on 0 / width / height and Z <= 0 are
    out; just inside is in."""
    px = [(0.0, 100.0), (640.0, 100.0), (100.0, 0.0), (100.0, 480.0), (0.5, 100.0), (639.5, 479.5), (200.0, 200.0)]
    X = np.array([back(u, v) for u, v in px] + [np.array([0.1, 0.1, 0.0]), np.array([0.1, 0.1, -2.0])])
    d = descs(len(X), 1)
    kf = points_frame(np.array(px + [(300.0, 300.0), (300.0, 300.0)]), d, with_P=False)
    lmap = dict(pt_X=X, pt_desc=d, ls_X=np.zeros((0, 6)), ls_desc=np.zeros((0, 32)))
    lm, n, _, _ = kfm.match_map2kf(CAM, prm(min_pt_matches=1), lmap, I4, kf, fast_matching=False)
    assert list(lm) == [-1, -1, -1, -1, 4, 5, 6, -1, -1] and n == 3


def test_kf2kf_query_lines_stay_in_pixels():
    """matchKF2KFLines leaves pj_lines in pixels (:392-393): a previous line projecting near the image origin lands in the
    window of a current line ten times further out (cells = pixels / 10 here), the others find no candidate."""
    d = descs(4, 2)
    prev = lines_frame([(10, 10, 20, 12), (300, 300, 400, 320), (350, 100, 450, 110), (200, 400, 260, 300)], d)
    curr = lines_frame([(100, 100, 200, 120), (300, 300, 400, 320), (350, 100, 450, 110), (200, 400, 260, 300)], d)
    _, _, m_ls, n_ls = kfm.match_kf2kf(CAM, prm(min_ls_matches=0), prev, curr, I4)
    assert list(m_ls) == [0, -1, -1, -1] and n_ls == 1
    # fewer than min_ls_matches windowed matches with more than min_ls_matches lines in both keyframes: match() for all
    _, _, m_ls, n_ls = kfm.match_kf2kf(CAM, prm(min_ls_matches=2), prev, curr, I4)
    assert list(m_ls) == [0, 1, 2, 3] and n_ls == 4


def test_fallback_conditions():
    d = descs(6, 3)
    px = [(50, 50), (150, 60), (250, 300), (400, 100), (500, 400), (600, 200)]
    far = [(x + 200 if x < 400 else x - 300, y) for x, y in px]        # nowhere near the projections: windowed finds nothing
    prev, curr = points_frame(px, d), points_frame(far, d)
    # KF-to-KF: n_curr > min && n_prev > min && matches < min (:274-276)
    m, n, _, _ = kfm.match_kf2kf(CAM, prm(min_pt_matches=5, matching_f2f_ws=0), prev, curr, I4)
    assert n == 6 and np.array_equal(m, np.arange(6))
    m, n, _, _ = kfm.match_kf2kf(CAM, prm(min_pt_matches=6, matching_f2f_ws=0), prev, curr, I4)   # 6 features, not > 6
    assert n == 0 and (m == -1).all()
    m, n, _, _ = kfm.match_kf2kf(CAM, prm(min_pt_matches=5, matching_f2f_ws=0), prev, points_frame(far[:5], d[:5]), I4)
    assert n == 0 and (m == -1).all()                                   # n_curr = 5, not > 5
    # map-to-KF: the visible-landmark count is tested twice (:594-595); the unmatched count (2 here) never is
    kf = points_frame(far, d, with_P=False)
    lmap = dict(pt_X=prev["pt_P"], pt_desc=d, ls_X=np.zeros((0, 6)), ls_desc=np.zeros((0, 32)))
    lm_mask = np.array([7, 7, 7, 7, -1, -1])
    lm, n, _, _ = kfm.match_map2kf(CAM, prm(min_pt_matches=5, matching_f2f_ws=0), lmap, I4, kf, kf_pt_lm=lm_mask,
                                   max_kf_epip_p=1e9)
    assert list(lm) == [-1, -1, -1, -1, 4, 5] and n == 2


def test_no_fast_matching_and_too_few_features_gives_nothing():
    d = descs(3, 4)
    f = points_frame([(100, 100), (200, 200), (300, 300)], d)
    m, n, _, _ = kfm.match_kf2kf(CAM, prm(min_pt_matches=10), f, f, I4, fast_matching=False)
    assert n == 0 and (m == -1).all()
    m, n, _, _ = kfm.match_kf2kf(CAM, prm(min_pt_matches=10), f, f, I4, fast_matching=True)
    assert n == 3 and np.array_equal(m, np.arange(3))
    m, n, _, _ = kfm.match_kf2kf(CAM, prm(min_pt_matches=2), f, f, I4, fast_matching=False)
    assert n == 3 and np.array_equal(m, np.arange(3))


def test_signed_line_gate_and_match_count():
    """le . (p, 1) < max_kf_epip_l without abs (:727-729): a large negative error passes; each reject decrements the
    return value (:748)."""
    d = descs(4, 5)
    kf = lines_frame([(100, 300, 500, 300), (100, 300, 500, 300), (100, 200, 500, 200), (100, 100, 500, 100)], d)
    # landmark 0: 200 px above its feature's line (error -200: passes), 1: 100 px below (+100: rejected), 2, 3: on the line
    Xl = [np.concatenate([back(150, 100), back(450, 100)]), np.concatenate([back(150, 400), back(450, 400)]),
          np.concatenate([back(150, 200), back(450, 200)]), np.concatenate([back(150, 100), back(450, 100)])]
    lmap = dict(pt_X=np.zeros((0, 3)), pt_desc=np.zeros((0, 32)), ls_X=np.array(Xl), ls_desc=d)
    _, _, lm, n = kfm.match_map2kf(CAM, prm(min_ls_matches=1), lmap, I4, kf, fast_matching=False)
    assert list(lm) == [0, -1, 2, 3] and n == 3          # 4 matches - 1 reject
    _, _, lm, n = kfm.match_map2kf(CAM, prm(min_ls_matches=1), lmap, I4, kf, fast_matching=False, max_kf_epip_l=-150.0)
    assert list(lm) == [0, -1, -1, -1] and n == 1


def test_point_gate_and_masks():
    """use = 0 landmarks and already matched keyframe features take no part; compact indices map back to original ones;
    |pf_map - pl| < max_kf_epip_p rejects (:612-613, :628)."""
    d = descs(6, 6)
    px = np.array([(100, 100), (200, 150), (300, 200), (400, 250), (500, 300), (600, 350)], np.float64)
    X = np.array([back(u, v) for u, v in px])
    kf_px = px.copy()
    kf_px[3] += (0.6, 0.8)                                             # 1.0 px away: not < 1.0
    kf_px[4] += (0.3, 0.4)
    kf = points_frame(kf_px, d, with_P=False)
    lmap = dict(pt_X=X, pt_desc=d, pt_use=np.array([1, 0, 1, 1, 1, 1], np.uint8), ls_X=np.zeros((0, 6)), ls_desc=np.zeros((0, 32)))
    lm, n, _, _ = kfm.match_map2kf(CAM, prm(min_pt_matches=1), lmap, I4, kf, kf_pt_lm=np.array([-1, -1, -1, -1, -1, 9]),
                                   fast_matching=False)
    assert list(lm) == [0, -1, 2, -1, 4, -1] and n == 3   # 4 pairs (landmark 5's feature is taken) - 1 reject


def test_kf2kf_points_at_identity_equal_pipeline_tracking():
    """With DT = I and fast_matching the KF-to-KF points are the pipeline's windowed tracking (oracle/frontend.py
    track_matches with matching_strategy != 0)."""
    rng = np.random.default_rng(7)
    n = 300
    px = np.stack([rng.uniform(5, 635, n), rng.uniform(5, 475, n)], 1)
    P = np.array([back(u, v, Z) for (u, v), Z in zip(px, rng.uniform(2, 30, n))])
    protos = rng.integers(0, 256, (40, 32), dtype=np.uint8)
    dp = protos[rng.integers(0, 40, n)] ^ np.packbits(rng.random((n, 256)) < 0.08, axis=1)
    perm = rng.permutation(n)[:250]
    curr_px = px[perm] + rng.normal(0, 6, (250, 2))
    dc = dp[perm] ^ np.packbits(rng.random((250, 256)) < 0.05, axis=1)
    prev = ofe.Frame(pt_P=P, pdesc=dp)
    curr = ofe.Frame(pt_pl=curr_px, pdesc=dc)
    for ws, kmin in ((3, 10), (1, 10), (0, 500)):
        p = prm(matching_strategy=3, matching_f2f_ws=ws, min_pt_matches=kmin)
        mp, _ = ofe.track_matches(CAM, prev, curr, p)
        m, cnt, _, _ = kfm.match_kf2kf(CAM, p, dict(pt_P=P, pdesc=dp, ldesc=np.zeros((0, 32), np.uint8)),
                                       dict(pt_pl=curr_px, pdesc=dc, ldesc=np.zeros((0, 32), np.uint8)), I4)
        assert np.array_equal(m, mp) and cnt == int((m >= 0).sum()) and cnt > 0


def test_clipped_walk_equals_full_walk():
    """The query walk restricted to the steps whose window reaches the grid visits exactly the cells of the full walk that
    can return a candidate."""
    from oracle import matchgrid as mg
    rng = np.random.default_rng(9)
    for _ in range(300):
        x1, y1, x2, y2 = rng.integers(-300, 400, 4)
        ws = int(rng.integers(0, 4))
        w = (ws, ws, ws, ws)
        keep = lambda c: c[0] + ws >= 0 and c[0] - ws < 64 and c[1] + ws >= 0 and c[1] - ws < 48
        full = [c for c in mg.bresenham(x1, y1, x2, y2) if keep(c)]
        clipped = [c for c in kfm._walk_clipped(x1, y1, x2, y2, w) if keep(c)]
        assert full == clipped
