"""Seeded synthetic stereo imagery (SURVEY.md §8d C1..C5): the input generator of bench.py and of the tests.
It is data generation only - no part of the hot path and no part of the CPU oracle (it imports neither).

scene_pair(): the C1 "plumbing" pair — filled random-gray rectangles + thin lines on gray 90, 3x3
sigma-0.8 blur, +-3 uniform noise, right image = left shifted by a constant disparity.
Stream rendering (planted SE(3) trajectory through a 3-D world of textured quads and segments) is in
world_* below.  Drawing uses cv2 (python OpenCV is part of the image on both the build container and
the GPU box); everything is deterministic given the seed.
"""
import math

import cv2
import numpy as np


def expmap_se3(x):
    """x = [t; w] -> 4x4 (SURVEY Appendix A.4), same operation order as the oracle's C helper."""
    x = np.asarray(x, np.float64)
    R = np.eye(3)
    t = x[:3].copy()
    w = x[3:]
    theta = math.sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2])
    if not (theta < 0.000001):
        s = np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]]) / theta
        s2 = np.empty((3, 3))
        for i in range(3):
            for j in range(3):
                s2[i, j] = s[i, 0] * s[0, j] + s[i, 1] * s[1, j] + s[i, 2] * s[2, j]
        sn, cs = math.sin(theta), math.cos(theta)
        I = np.eye(3)
        R = I + s * sn + s2 * (1.0 - cs)
        V = I + s * (1.0 - cs) / theta + s2 * (theta - sn) / theta
        t = np.array([V[i, 0] * t[0] + V[i, 1] * t[1] + V[i, 2] * t[2] for i in range(3)])
    T = np.eye(4)
    T[:3, :3] = R
    T[:3, 3] = t
    return T


def scene_pair(w=1242, h=375, seed=1, n_rect=220, n_lines=120, disparity=20, noise=3):
    rng = np.random.default_rng(seed)
    W = w + disparity
    img = np.full((h, W), 90, np.uint8)
    for _ in range(n_rect):
        x0 = int(rng.integers(-40, W)); y0 = int(rng.integers(-40, h))
        rw = int(rng.integers(12, 160)); rh = int(rng.integers(10, 110))
        g = int(rng.integers(20, 236))
        cv2.rectangle(img, (x0, y0), (x0 + rw, y0 + rh), g, -1)
    for _ in range(n_lines):
        p0 = (int(rng.integers(0, W)), int(rng.integers(0, h)))
        ang = rng.uniform(0, np.pi); L = rng.uniform(30, 300)
        p1 = (int(p0[0] + L * np.cos(ang)), int(p0[1] + L * np.sin(ang)))
        cv2.line(img, p0, p1, int(rng.integers(0, 256)), int(rng.integers(1, 3)), cv2.LINE_8)
    img = cv2.GaussianBlur(img, (3, 3), 0.8)
    def noisy(a, r):
        n = r.integers(-noise, noise + 1, a.shape)
        return np.clip(a.astype(np.int16) + n, 0, 255).astype(np.uint8)
    left = noisy(img[:, 0:w], rng)                       # x_left = x_right + disparity
    right = noisy(img[:, disparity:disparity + w], rng)
    return np.ascontiguousarray(left), np.ascontiguousarray(right)


# ---- synthetic correspondences for the pose optimiser (SURVEY §4 item 3: planted pose) ---------------
def project(cam, P):
    P = np.asarray(P, np.float64)
    return np.stack([cam["cx"] + cam["fx"] * P[:, 0] / P[:, 2], cam["cy"] + cam["fy"] * P[:, 1] / P[:, 2]], 1)


def gn_problem(cam, n_pts=300, n_lines=80, seed=0, x_true=None, px_noise=0.3, outlier_frac=0.1, z_range=(4, 40)):
    """3-D points / segments in the previous camera frame (depths uniform in z_range) + their observations in the
    current frame under a planted increment T_true (current <- previous), with pixel noise and gross outliers."""
    rng = np.random.default_rng(seed)
    if x_true is None:
        x_true = np.array([0.05, -0.02, 0.9, 0.01, -0.03, 0.005])
    T = expmap_se3(x_true)
    def rand_pts(n):
        z = rng.uniform(z_range[0], z_range[1], n)
        u = rng.uniform(30, cam["width"] - 30, n); v = rng.uniform(20, cam["height"] - 20, n)
        return np.stack([(u - cam["cx"]) * z / cam["fx"], (v - cam["cy"]) * z / cam["fy"], z], 1)
    P = rand_pts(n_pts)
    Pc = P @ T[:3, :3].T + T[:3, 3]
    obs = project(cam, Pc) + rng.normal(0, px_noise, (n_pts, 2))
    n_out = int(outlier_frac * n_pts)
    obs[:n_out] += rng.uniform(-60, 60, (n_out, 2))
    sP = rand_pts(n_lines)
    eP = sP + rng.normal(0, 1.0, (n_lines, 3)) * np.array([1.5, 1.0, 0.5])
    eP[:, 2] = np.maximum(eP[:, 2], 2.0)
    sp = project(cam, sP @ T[:3, :3].T + T[:3, 3]) + rng.normal(0, px_noise, (n_lines, 2))
    ep = project(cam, eP @ T[:3, :3].T + T[:3, 3]) + rng.normal(0, px_noise, (n_lines, 2))
    n_outl = int(outlier_frac * n_lines)
    sp[:n_outl] += rng.uniform(-40, 40, (n_outl, 2))
    sph = np.concatenate([sp, np.ones((n_lines, 1))], 1); eph = np.concatenate([ep, np.ones((n_lines, 1))], 1)
    le = np.cross(sph, eph)
    le = le / np.sqrt(le[:, 0:1] ** 2 + le[:, 1:2] ** 2)      # le = (sp x ep) / ||(le0, le1)||  (SURVEY a6)
    return dict(P=P, obs=obs, sP=sP, eP=eP, le=le, T_true=T, x_true=np.asarray(x_true, np.float64))


# ---- synthetic stereo streams with a planted SE(3) trajectory (SURVEY §8d C2..C5) ------------------------------
class World:
    """Fronto-parallel textured quads (random-checker albedo) + 3-D line segments along a corridor in +z."""

    def __init__(self, seed=7, length=120.0, n_quads=260, n_segs=140, albedo_sigma=60.0, cells=4,
                 half_width=14.0, half_height=4.5):
        rng = np.random.default_rng(seed)
        self.quads = []   # (centre xyz, half sizes, cell grays [cells x cells])
        for _ in range(n_quads):
            z = rng.uniform(4.0, length)
            side = rng.choice([-1.0, 1.0])
            x = side * rng.uniform(1.2, half_width)
            y = rng.uniform(-half_height, half_height * 0.6)
            hw, hh = rng.uniform(0.4, 2.2), rng.uniform(0.3, 1.6)
            base = rng.uniform(40, 215)
            g = np.clip(base + rng.normal(0, albedo_sigma, (cells, cells)), 5, 250)
            self.quads.append((np.array([x, y, z]), hw, hh, g))
        self.segs = []
        for _ in range(n_segs):
            z = rng.uniform(4.0, length)
            x = rng.uniform(-half_width, half_width); y = rng.uniform(-half_height, half_height)
            d = rng.normal(0, 1, 3) * np.array([2.0, 1.2, 0.3])
            self.segs.append((np.array([x, y, z]), np.array([x, y, z]) + d, float(rng.uniform(10, 245)), int(rng.integers(1, 3))))
        self.cells = cells


def corridor_world(n_segs=450, seed=3):
    """Lines-dominant scene (BASELINE configs[4]): long low-contrast 3-D segments running along the corridor (few
    crossings, ends mostly outside the view), no textured quads."""
    world = World(seed=21, length=90.0, n_quads=0, n_segs=0)
    rng = np.random.default_rng(seed)
    segs = []
    for _ in range(n_segs):
        x = rng.choice([-1, 1]) * rng.uniform(1.0, 12.0); y = rng.uniform(-4, 4)
        z0 = rng.uniform(1.0, 30.0); z1 = z0 + rng.uniform(15, 60)
        g = float(90 + rng.choice([-1, 1]) * rng.uniform(24, 32))
        segs.append((np.array([x, y, z0]), np.array([x + rng.normal(0, 0.05), y + rng.normal(0, 0.05), z1]), g, int(rng.integers(2, 4))))
    world.segs = segs
    return world


def _project(cam, Pc):
    return np.stack([cam["cx"] + cam["fx"] * Pc[:, 0] / Pc[:, 2], cam["cy"] + cam["fy"] * Pc[:, 1] / Pc[:, 2]], 1)


def render_view(world, cam, T_cw, x_offset=0.0, noise_rng=None, noise=3, bg=90):
    """Renders one camera view. T_cw: camera <- world (4x4). x_offset: camera-frame x shift (right eye = +b)."""
    w, h = cam["width"], cam["height"]
    img = np.full((h, w), bg, np.uint8)
    R, t = T_cw[:3, :3], T_cw[:3, 3].copy()
    t[0] -= x_offset
    items = []
    for (c, hw, hh, g) in world.quads:
        zc = (R @ c + t)[2]
        if 1.0 < zc < 90.0:
            items.append((zc, 0, (c, hw, hh, g)))
    for (a, b, gray, th) in world.segs:
        za, zb = (R @ a + t)[2], (R @ b + t)[2]
        if za > 1.0 and zb > 1.0 and min(za, zb) < 90.0:
            items.append((max(za, zb), 1, (a, b, gray, th)))
    items.sort(key=lambda it: -it[0])     # painter's algorithm: far to near
    SH = 4
    for _, kind, it in items:
        if kind == 0:
            c, hw, hh, g = it
            n = g.shape[0]
            xs = np.linspace(-hw, hw, n + 1); ys = np.linspace(-hh, hh, n + 1)
            gx, gy = np.meshgrid(xs, ys)
            Pw = np.stack([c[0] + gx.ravel(), c[1] + gy.ravel(), np.full(gx.size, c[2])], 1)
            Pc = Pw @ R.T + t
            if (Pc[:, 2] < 0.5).any():
                continue
            uv = _project(cam, Pc).reshape(n + 1, n + 1, 2)
            if uv[..., 0].max() < -50 or uv[..., 0].min() > w + 50 or uv[..., 1].max() < -50 or uv[..., 1].min() > h + 50:
                continue
            for i in range(n):
                for j in range(n):
                    poly = np.array([uv[i, j], uv[i, j + 1], uv[i + 1, j + 1], uv[i + 1, j]])
                    cv2.fillConvexPoly(img, np.round(poly * (1 << SH)).astype(np.int32), int(g[i, j]), cv2.LINE_AA, SH)
        else:
            a, b, gray, th = it
            Pc = np.stack([a, b]) @ R.T + t
            uv = _project(cam, Pc)
            if np.abs(uv).max() > 1e5:
                continue
            p0 = tuple(int(v) for v in np.round(uv[0] * (1 << SH))); p1 = tuple(int(v) for v in np.round(uv[1] * (1 << SH)))
            cv2.line(img, p0, p1, int(gray), th, cv2.LINE_AA, SH)
    img = cv2.GaussianBlur(img, (3, 3), 0.8)
    if noise_rng is not None and noise > 0:
        img = np.clip(img.astype(np.int16) + noise_rng.integers(-noise, noise + 1, img.shape), 0, 255).astype(np.uint8)
    return img


def trajectory(n_frames, seed=42, step=0.4, yaw_deg=0.6, lateral=0.02):
    """Planted camera poses T_wc (world <- camera): forward motion with small yaw / lateral jitter."""
    rng = np.random.default_rng(seed)
    T = np.eye(4)
    out = [T.copy()]
    for _ in range(n_frames - 1):
        x = np.array([rng.normal(0, lateral), rng.normal(0, lateral * 0.5), step * rng.uniform(0.8, 1.2),
                      np.deg2rad(rng.normal(0, yaw_deg * 0.3)), np.deg2rad(rng.normal(0, yaw_deg)), np.deg2rad(rng.normal(0, yaw_deg * 0.2))])
        T = T @ expmap_se3(x)
        out.append(T.copy())
    return out


def stream(cam, n_frames, world=None, seed=42, traj=None, noise=3, **traj_kw):
    """Yields (left, right, T_wc) for a planted trajectory.  Right camera is offset by the baseline along +x."""
    world = world or World()
    traj = traj or trajectory(n_frames, seed=seed, **traj_kw)
    rng = np.random.default_rng(seed + 1000)
    for T_wc in traj:
        T_cw = np.linalg.inv(T_wc)
        L = render_view(world, cam, T_cw, 0.0, rng, noise)
        Rr = render_view(world, cam, T_cw, cam["b"], rng, noise)
        yield L, Rr, T_wc


# ---- synthetic local-map problems for the bundle adjustment (SURVEY 8(f) f4) ------------------------------------
def _logmap_se3(T):
    """logmap_se3 (SURVEY Appendix A.4), numpy; x = [t; w]."""
    R, t = T[:3, :3], T[:3, 3]
    c = min(1.0, max(-1.0, (np.trace(R) - 1.0) / 2.0))
    theta = math.acos(c)
    w = np.zeros(3)
    V = np.eye(3)
    if theta > 1e-6:
        sn = math.sqrt(max(0.0, 1.0 - c * c))
        W = (R - R.T) * (theta / (2.0 * sn))
        w = np.array([W[2, 1], W[0, 2], W[1, 0]])
        s = np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]]) / theta
        V = np.eye(3) + s * (1.0 - c) / theta + (s @ s) * (theta - sn) / theta
    return np.concatenate([np.linalg.solve(V, t), w])


def lba_problem(cam, n_kf=4, n_fixed=2, n_pt=120, n_ls=40, seed=0, px_noise=0.3, pose_noise=0.01, lm_noise=0.02):
    """A local map as MapHandler::localBundleAdjustment assembles it (src/mapHandler.cpp:1220-1330): n_kf local keyframes
    (optimised) + n_fixed fixed ones along a forward trajectory, point and line landmarks in front of them, every landmark
    observed by the keyframes that see it (observations grouped per landmark, as the reference builds its lists).  Poses
    are T_kf_w (keyframe -> world) as se(3) vectors; the returned initial values are perturbed copies of the truth."""
    rng = np.random.default_rng(seed)
    poses = []
    for i in range(n_kf + n_fixed):
        x = np.array([0.05 * rng.standard_normal(), 0.02 * rng.standard_normal(), 0.8 * i, 0.01 * rng.standard_normal(),
                      0.03 * rng.standard_normal(), 0.005 * rng.standard_normal()])
        poses.append(expmap_se3(x))
    fixed_T = np.stack(poses[:n_fixed]) if n_fixed else np.zeros((0, 4, 4))
    local_T = poses[n_fixed:]

    def rand_world(n):
        z = rng.uniform(6, 40, n) + 0.8 * (n_kf + n_fixed)
        u = rng.uniform(60, cam["width"] - 60, n); v = rng.uniform(40, cam["height"] - 40, n)
        return np.stack([(u - cam["cx"]) * (z - 4) / cam["fx"], (v - cam["cy"]) * (z - 4) / cam["fy"], z], 1)

    def view(T_kf_w, Pw):
        Ti = np.linalg.inv(T_kf_w)
        Pc = Pw @ Ti[:3, :3].T + Ti[:3, 3]
        uv = np.stack([cam["cx"] + cam["fx"] * Pc[:, 0] / Pc[:, 2], cam["cy"] + cam["fy"] * Pc[:, 1] / Pc[:, 2]], 1)
        ok = (Pc[:, 2] > 1.0) & (uv[:, 0] > 0) & (uv[:, 0] < cam["width"]) & (uv[:, 1] > 0) & (uv[:, 1] < cam["height"])
        return uv, ok

    pt = rand_world(n_pt)
    a = rand_world(n_ls)
    ls = np.concatenate([a, a + rng.uniform(-2.0, 2.0, (n_ls, 3)) * np.array([1.0, 0.5, 0.3])], 1)
    all_T = [(-1 - k, fixed_T[k]) for k in range(n_fixed)] + [(k, local_T[k]) for k in range(n_kf)]
    po_lm, po_kf, po_xy, lo_lm, lo_kf, lo_le = [], [], [], [], [], []
    # (a landmark nobody observes would leave a zero block in the Hessian: the first keyframe always keeps its observation)
    for j in range(n_pt):
        for i, (kf, T) in enumerate(all_T):
            uv, ok = view(T, pt[j:j + 1])
            if i == 0 or (ok[0] and rng.uniform() < 0.8):
                po_lm.append(j); po_kf.append(kf); po_xy.append(uv[0] + px_noise * rng.standard_normal(2))
    for j in range(n_ls):
        for i, (kf, T) in enumerate(all_T):
            s, oks = view(T, ls[j:j + 1, :3]); e, oke = view(T, ls[j:j + 1, 3:])
            if i == 0 or (oks[0] and oke[0] and rng.uniform() < 0.8):
                sp = np.append(s[0] + px_noise * rng.standard_normal(2), 1.0); ep = np.append(e[0] + px_noise * rng.standard_normal(2), 1.0)
                le = np.cross(sp, ep)
                lo_lm.append(j); lo_kf.append(kf); lo_le.append(le / math.sqrt(le[0] * le[0] + le[1] * le[1]))
    kf_true = np.stack([_logmap_se3(T) for T in local_T]) if n_kf else np.zeros((0, 6))
    return dict(kf_pose=kf_true + pose_noise * rng.standard_normal(kf_true.shape), pt=pt + lm_noise * rng.standard_normal(pt.shape),
                ls=ls + lm_noise * rng.standard_normal(ls.shape), fixed_T=fixed_T,
                pt_obs_lm=np.array(po_lm, np.int32), pt_obs_kf=np.array(po_kf, np.int32), pt_obs_xy=np.array(po_xy).reshape(-1, 2),
                ls_obs_lm=np.array(lo_lm, np.int32), ls_obs_kf=np.array(lo_kf, np.int32), ls_obs_le=np.array(lo_le).reshape(-1, 3),
                truth=dict(kf_pose=kf_true, pt=pt, ls=ls))


def local_map_problem(cam, n_kf=8, n_fixed=2, pts_per_kf=6, ls_per_kf=2, seed=0, t0=0, single=0.3, max_track=3,
                      px_noise=0.3, pose_noise=0.01, lm_noise=0.02):
    """A local map shaped like the ones MapHandler::localBundleAdjustment assembles (src/mapHandler.cpp:1220-1330), from
    a sliding window of n_fixed fixed keyframes followed by n_kf local ones, 0.8 m apart along the optical axis.  The
    window starts at keyframe t0 of the trajectory, whose keyframe 0 is the world frame: with t0 = 0 the first fixed
    keyframe (fixed_T[0]) is the identity, otherwise no keyframe is.
    Every keyframe of the window creates pts_per_kf points and ls_per_kf lines that only it and the next k keyframes
    observe.  A fraction `single` of the landmarks (rounded) has k = 0, one observation: all those the last keyframe
    creates (it creates fewer when the window is too short for that to stay within `single`) and others drawn at
    random.  The rest have k uniform in 1..max_track, cut at the window's end.  So some landmarks are seen by local
    keyframes only, some by fixed ones only, and the fixed keyframes observe landmarks the local ones see too.
    Observations are grouped per landmark in ascending order, creator first; kf_obs is the local index, or -1 - k for
    fixed_T[k].  Observations are the true projections plus px_noise; the initial values are the truth plus pose_noise
    / lm_noise.  truth holds the window's poses T_kf_w (fixed first) and the true landmarks."""
    rng = np.random.default_rng(seed)
    n_tot = n_kf + n_fixed
    T = []
    for i in range(n_tot):
        t = t0 + i
        x = np.zeros(6) if t == 0 else np.array([0.05 * rng.standard_normal(), 0.02 * rng.standard_normal(), 0.8 * t,
                                                   0.01 * rng.standard_normal(), 0.03 * rng.standard_normal(),
                                                   0.005 * rng.standard_normal()])
        T.append(np.eye(4) if t == 0 else expmap_se3(x))
    T = np.stack(T)
    Ti = np.linalg.inv(T)
    kf_id = lambda t: -1 - t if t < n_fixed else t - n_fixed

    def counts(per):   # landmarks created by each keyframe: the last one's are all single
        c = np.full(n_tot, per)
        if n_tot > 1:
            c[-1] = min(per, int(single * (n_tot - 1) * per / (1.0 - single)))
        return c

    def tracks(creator):   # k per landmark
        n = len(creator)
        k = np.minimum(rng.integers(1, max_track + 1, n), n_tot - 1 - creator)
        forced = k == 0
        extra = max(0, int(round(single * n)) - int(forced.sum()))
        pick = rng.choice(np.flatnonzero(~forced), min(extra, int((~forced).sum())), replace=False)
        k[pick] = 0
        return k

    def in_front(creator):   # a point 6-30 m ahead of its creator, within the middle of the image
        z = rng.uniform(6.0, 30.0, len(creator))
        u = rng.uniform(0.3, 0.7, len(creator)) * cam["width"]; v = rng.uniform(0.3, 0.7, len(creator)) * cam["height"]
        Pc = np.stack([(u - cam["cx"]) * z / cam["fx"], (v - cam["cy"]) * z / cam["fy"], z, np.ones_like(z)], 1)
        return np.einsum("nij,nj->ni", T[creator], Pc)[:, :3]

    def project(t, P):
        Pc = Ti[t, :3, :3] @ P + Ti[t, :3, 3]
        return np.array([cam["cx"] + cam["fx"] * Pc[0] / Pc[2], cam["cy"] + cam["fy"] * Pc[1] / Pc[2]])

    pc = np.repeat(np.arange(n_tot), counts(pts_per_kf))
    lc = np.repeat(np.arange(n_tot), counts(ls_per_kf))
    pt = in_front(pc)
    ls = np.concatenate([in_front(lc), in_front(lc)], 1)
    pk, lk = tracks(pc), tracks(lc)
    po_lm, po_kf, po_xy, lo_lm, lo_kf, lo_le = [], [], [], [], [], []
    for j in range(len(pt)):
        for t in range(pc[j], pc[j] + pk[j] + 1):
            po_lm.append(j); po_kf.append(kf_id(t)); po_xy.append(project(t, pt[j]) + px_noise * rng.standard_normal(2))
    for j in range(len(ls)):
        for t in range(lc[j], lc[j] + lk[j] + 1):
            s = np.append(project(t, ls[j, :3]) + px_noise * rng.standard_normal(2), 1.0)
            e = np.append(project(t, ls[j, 3:]) + px_noise * rng.standard_normal(2), 1.0)
            le = np.cross(s, e)
            lo_lm.append(j); lo_kf.append(kf_id(t)); lo_le.append(le / math.sqrt(le[0] * le[0] + le[1] * le[1]))
    kf_true = np.stack([_logmap_se3(T[t]) for t in range(n_fixed, n_tot)]) if n_kf else np.zeros((0, 6))
    return dict(kf_pose=kf_true + pose_noise * rng.standard_normal(kf_true.shape),
                pt=pt + lm_noise * rng.standard_normal(pt.shape), ls=ls + lm_noise * rng.standard_normal(ls.shape),
                fixed_T=T[:n_fixed].copy(),
                pt_obs_lm=np.array(po_lm, np.int32), pt_obs_kf=np.array(po_kf, np.int32),
                pt_obs_xy=np.array(po_xy, np.float64).reshape(-1, 2),
                ls_obs_lm=np.array(lo_lm, np.int32), ls_obs_kf=np.array(lo_kf, np.int32),
                ls_obs_le=np.array(lo_le, np.float64).reshape(-1, 3),
                truth=dict(T=T, kf_pose=kf_true, pt=pt, ls=ls))


def gba_problem(cam, n_kf=64, pts_per_kf=100, ls_per_kf=15, loop=True, seed=0, n_fixed=1, n_views=3, px_noise=0.3,
                pose_noise=0.01, lm_noise=0.02):
    """A whole map as MapHandler::globalBundleAdjustment assembles it (src/mapHandler.cpp:1995-2090): n_fixed fixed
    keyframes (keyframe 0 and any others held fixed) followed by n_kf optimised ones, in kf_idx order, on a circle of
    0.8 m steps (a full turn when there are 40 keyframes or more) with the camera facing the same way throughout.  Each keyframe creates pts_per_kf points and
    ls_per_kf lines in front of it; each landmark is observed by its creator and by the next n_views - 1 keyframes that
    see it, so the reduced system is banded.  With `loop`, the last n_views keyframes also re-observe the landmarks of
    the first ones where they see them (the loop closure).  Observations are grouped per landmark in ascending order;
    every landmark is observed (by its creator).  Vectorised: 4096 keyframes generate in seconds."""
    rng = np.random.default_rng(seed)
    n_tot = n_kf + n_fixed
    step = 0.8
    dth = 2.0 * math.pi / max(n_tot, 40)
    R = step / dth
    th = dth * np.arange(n_tot)
    # one heading throughout, 0.6 rad off the world axes: rotations near 0 or pi are where logmap_se3's acos loses digits
    yaw = 0.6 + 0.002 * rng.standard_normal(n_tot)
    c, s_ = np.cos(yaw), np.sin(yaw)
    Tw = np.zeros((n_tot, 4, 4))
    Tw[:, :3, 0] = np.stack([c, np.zeros_like(c), -s_], 1)       # right
    Tw[:, :3, 1] = [0.0, 1.0, 0.0]                               # down
    Tw[:, :3, 2] = np.stack([s_, np.zeros_like(c), c], 1)        # forward
    Tw[:, :3, 3] = np.stack([R * (1 - np.cos(th)), 0.05 * rng.standard_normal(n_tot), R * np.sin(th)], 1)
    Tw[:, 3, 3] = 1.0
    Ti = np.linalg.inv(Tw)

    def in_view(creators, n):
        z = rng.uniform(4.0, 20.0, n)
        u = rng.uniform(40, cam["width"] - 40, n); v = rng.uniform(30, cam["height"] - 30, n)
        Pc = np.stack([(u - cam["cx"]) * z / cam["fx"], (v - cam["cy"]) * z / cam["fy"], z], 1)
        return np.einsum("nij,nj->ni", Tw[creators, :3, :3], Pc) + Tw[creators, :3, 3]

    def project(t, Pw):   # t: [m] observer indices, Pw: [m, 3]
        Pc = np.einsum("nij,nj->ni", Ti[t, :3, :3], Pw) + Ti[t, :3, 3]
        with np.errstate(divide="ignore", invalid="ignore"):
            uv = np.stack([cam["cx"] + cam["fx"] * Pc[:, 0] / Pc[:, 2], cam["cy"] + cam["fy"] * Pc[:, 1] / Pc[:, 2]], 1)
        ok = (Pc[:, 2] > 1.0) & (uv[:, 0] > 0) & (uv[:, 0] < cam["width"]) & (uv[:, 1] > 0) & (uv[:, 1] < cam["height"])
        return uv, ok

    def observers(creators):   # [n, 2 n_views] candidate observer per landmark, -1 where none, creator first
        o = np.arange(n_views)
        fwd = creators[:, None] + o[None, :]
        fwd[fwd >= n_tot] = -1
        back = np.full_like(fwd, -1)
        if loop:
            b = (n_tot - 1 - o)[None, :].repeat(len(creators), 0)
            ok = (creators[:, None] < n_views) & (b > creators[:, None] + n_views - 1)
            back[ok] = b[ok]
        return np.concatenate([fwd, back], 1)

    def observe(cand, ends):   # -> (landmark index, observer, projections of each end point) of the kept candidates
        lm, col = np.nonzero(cand >= 0)
        t = cand[lm, col]
        uvs, ok = [], col == 0
        keep = np.ones(len(t), bool)
        for P in ends:
            uv, vis = project(t, P[lm])
            uvs.append(uv); keep &= vis
        keep |= ok
        return lm[keep], t[keep], [uv[keep] for uv in uvs]

    kf_of = lambda t: np.where(t < n_fixed, -1 - t, t - n_fixed).astype(np.int32)
    pc = np.repeat(np.arange(n_tot), pts_per_kf)
    pt = in_view(pc, len(pc))
    plm, pt_t, (puv,) = observe(observers(pc), [pt])
    lc = np.repeat(np.arange(n_tot), ls_per_kf)
    ls = np.concatenate([in_view(lc, len(lc)), in_view(lc, len(lc))], 1)
    llm, ls_t, (suv, euv) = observe(observers(lc), [ls[:, :3], ls[:, 3:]])
    sp = np.concatenate([suv + px_noise * rng.standard_normal(suv.shape), np.ones((len(suv), 1))], 1)
    ep = np.concatenate([euv + px_noise * rng.standard_normal(euv.shape), np.ones((len(euv), 1))], 1)
    le = np.cross(sp, ep)
    le /= np.hypot(le[:, 0], le[:, 1])[:, None]
    kf_true = np.stack([_logmap_se3(T) for T in Tw[n_fixed:]]) if n_kf else np.zeros((0, 6))
    # the initial poses are perturbed in each keyframe's own frame: noise added to the se(3) vector of a keyframe far
    # from the origin would move it by |t| times the rotation noise, metres on a long map
    noise = pose_noise * rng.standard_normal(kf_true.shape)
    kf_init = np.stack([_logmap_se3(T @ expmap_se3(e)) for T, e in zip(Tw[n_fixed:], noise)]) if n_kf else np.zeros((0, 6))
    return dict(kf_pose=kf_init,
                pt=pt + lm_noise * rng.standard_normal(pt.shape), ls=ls + lm_noise * rng.standard_normal(ls.shape),
                fixed_T=Tw[:n_fixed].copy(),
                pt_obs_lm=plm.astype(np.int32), pt_obs_kf=kf_of(pt_t), pt_obs_xy=puv + px_noise * rng.standard_normal(puv.shape),
                ls_obs_lm=llm.astype(np.int32), ls_obs_kf=kf_of(ls_t), ls_obs_le=le,
                truth=dict(kf_pose=kf_true, pt=pt, ls=ls))


def _rodrigues(w):
    """rotation matrices of the rotation vectors w [n, 3]"""
    w = np.asarray(w, np.float64).reshape(-1, 3)
    th = np.linalg.norm(w, axis=1)
    k = w / np.where(th > 0, th, 1.0)[:, None]
    K = np.zeros((len(w), 3, 3))
    K[:, 0, 1], K[:, 0, 2], K[:, 1, 2] = -k[:, 2], k[:, 1], -k[:, 0]
    K -= K.transpose(0, 2, 1)
    s, c = np.sin(th)[:, None, None], np.cos(th)[:, None, None]
    return np.eye(3) + s * K + (1.0 - c) * (K @ K)


def _iso(R, t):
    T = np.zeros((len(R), 4, 4))
    T[:, :3, :3], T[:, :3, 3], T[:, 3, 3] = R, t, 1.0
    return T


def _iso_inv(T):
    Rt = T[:, :3, :3].transpose(0, 2, 1)
    return _iso(Rt, -np.einsum("nij,nj->ni", Rt, T[:, :3, 3]))


def pose_graph_problem(n_kf=256, window=5, n_lc=2, drift=0.01, seed=0, step=0.5, lc_noise=1e-3):
    """A loop-closure pose graph as MapHandler::loopClosureOptimizationCovGraphG2O builds it (plf_pose_graph's layout).
    Ground truth: n_kf keyframes `step` apart on a closed loop (a circle with a vertical wave).  T (T_kf_w) integrates
    the true relative motions perturbed by `drift` (radians and `drift * step` metres, normal, per step) from keyframe 0,
    which is fixed.  kf2kf edges join every pair 1 <= j - i <= window in (i asc, j asc) order and measure T_i^-1 T_j of
    the drifted poses, as the reference measures its current poses; then n_lc loop edges from a keyframe near the start
    to one near the end measure the true relative pose perturbed by `lc_noise`.  Returns dict(T, T_true, fixed, from, to,
    Z) with T [n_kf, 4, 4], fixed [n_kf] uint8, from / to [n_e] int32 and Z [n_e, 4, 4]."""
    rng = np.random.default_rng(seed)
    n = int(n_kf)
    k = np.arange(n)
    r = n * step / (2.0 * math.pi)
    a = 2.0 * math.pi * k / n
    yaw = a + math.pi / 2.0
    p = np.stack([r * np.cos(a), r * np.sin(a), 0.5 * np.sin(3.0 * a)], 1)
    Rt = _rodrigues(np.stack([0.02 * np.sin(5.0 * a), 0.02 * np.cos(7.0 * a), yaw], 1) * [[1.0, 1.0, 0.0]]) @ \
        _rodrigues(np.stack([0 * a, 0 * a, yaw], 1))
    T_true = _iso(Rt, p)
    D = _iso_inv(T_true[:-1]) @ T_true[1:]                          # true relative motions
    N = _iso(_rodrigues(drift * rng.standard_normal((n - 1, 3))), drift * step * rng.standard_normal((n - 1, 3)))
    D = D @ N
    T = np.empty_like(T_true)
    T[0] = T_true[0]
    for i in range(1, n):
        T[i] = T[i - 1] @ D[i - 1]
    ii, dd = np.meshgrid(k, np.arange(1, window + 1), indexing="ij")
    jj = ii + dd
    keep = jj < n
    frm, to = ii[keep], jj[keep]
    Z = _iso_inv(T[frm]) @ T[to]
    if n_lc:
        la = np.arange(n_lc) * max(1, window // 2 + 1)
        lb = n - 1 - np.arange(n_lc) * max(1, window // 2 + 1)
        ok = lb > la + window
        la, lb = la[ok], lb[ok]
        Zl = _iso_inv(T_true[la]) @ T_true[lb] @ _iso(_rodrigues(lc_noise * rng.standard_normal((len(la), 3))),
                                                    lc_noise * rng.standard_normal((len(la), 3)))
        frm, to, Z = np.concatenate([frm, la]), np.concatenate([to, lb]), np.concatenate([Z, Zl])
    fixed = np.zeros(n, np.uint8)
    fixed[0] = 1
    return dict(T=T, T_true=T_true, fixed=fixed, **{"from": frm.astype(np.int32)}, to=to.astype(np.int32), Z=Z)
