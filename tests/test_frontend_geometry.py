"""The image geometries the front-end's tile kernels treat differently, and a model of their index arithmetic (CPU).

Every tile kernel of ORB, LSD and the LBD prelude stages its tile plus halo with one TMA box that must start on a
16-byte boundary, so the tile grids are shifted (plf_tma.cuh): FAST loads a 96 x 38 box from the aligned address at or
below x0 - 4, the blurs place their tiles at 64 bx - (16 - R) (plf_tma_tiles_x), and border CTAs rebuild
BORDER_REFLECT_101 in shared memory (plf_tma_reflect_fix), skipping mirror cells outside the box.  k_resize_exact4 reads
whole 32-bit words from a packed x table padded to a multiple of four columns.  Whether each of these is right depends
on w mod 16 / 62 / 64, h mod 16 / 30 / 32 and the pyramid level sizes, so this module:

  - builds the sweep of shapes (widths, heights, ORB base sizes) from the kernels' own tile constants, read from the
    #defines in csrc/*.cu, so that a retiled kernel is tested at its new edges (tests/test_frontend_geometry_gpu.py runs
    the detectors over it on the device);
  - checks that the sweep covers every residue and boundary it is meant to;
  - models the box origins, the tile grids and plf_tma_reflect_fix in Python for every shape of the sweep and asserts
    that every cell an output reads holds the BORDER_REFLECT_101 pixel it should;
  - checks the resize tables of the library itself (host code, no device needed) against the k_resize_exact4 window;
  - compares the C restatements clib.orb / clib.lsd with cv2 at the tiny and boundary shapes."""
import ctypes as C
import math
import re
from pathlib import Path

import numpy as np
import pytest

from param_cases import LSD_CASES, ORB_CASES, lsd_ksize, lsd_pre_ks

CSRC = Path(__file__).resolve().parent.parent / "pl-slam_b200" / "csrc"
TILE_NAMES = ("FN_OW", "FN_OH", "OBF_TW", "OBF_TH", "ORB_TW", "ORB_TH", "BF_TW", "BF_TH", "BQ_TW", "BQ_TH",
              "LBF_TW", "LBF_TH", "LBD_TW", "LBD_TH", "LSD_SEG", "LSD_PRE_TH", "LSD_PRE_BOXW", "LSD_PRE_BOXH", "LSD_PRE_HW",
              "LSD_PRE_KS_MAX")


def tile_consts():
    """{name: value} of the tile #defines of csrc/*.cu."""
    out = {}
    for f in sorted(CSRC.glob("*.cu")):
        for name, val in re.findall(r"^#define\s+(\w+)\s+(\d+)\b", f.read_text(), re.M):
            if name in TILE_NAMES:
                out[name] = int(val)
    assert set(out) == set(TILE_NAMES), set(TILE_NAMES) - set(out)
    return out


T = tile_consts()
ORB_BLUR_R = 3                       # k_orb_blur7_fast: 7 x 7 Gaussian
LBD_R = 3                            # k_blur5_sobel_fast: 5 x 5 blur + 3 x 3 Sobel
LSD_RADII = sorted({lsd_ksize(c) // 2 for c in [{}, *LSD_CASES.values()] if lsd_ksize(c)})
ORB_MIN_EDGE = 19


# ---- the kernels' grids ------------------------------------------------------------------------------------------
def tma_tiles_x(w, r):
    """plf_tma_tiles_x"""
    return (w + (16 - r) + 63) // 64


# shifted TMA blur tiles: (tile width, tile height, box width RP, columns read NEED, radius)
def shifted_kernels():
    return {"orb_blur7": (T["OBF_TW"], T["OBF_TH"], 80, 72, ORB_BLUR_R), "lbd_blur5_sobel": (T["LBF_TW"], T["LBF_TH"], 80, 76, LBD_R)}


def reflect101(i, n):
    """plf_reflect101, vectorised"""
    i = np.asarray(i, np.int64).copy()
    if n == 1:
        return np.zeros_like(i)
    while True:
        lo, hi = i < 0, i >= n
        if not (lo.any() or hi.any()):
            return i
        i[lo] = -i[lo]
        hi = i >= n
        i[hi] = 2 * (n - 1) - i[hi]


def reflect_fix_model(gx0, gy0, w, h, RH, RP, need_w):
    """The box after plf_tma_tiles' load and plf_tma_reflect_fix: raw[ry][rx] = the linear index of the image pixel the
    cell holds, -1 for a zero-filled cell (outside the image)."""
    gx = gx0 + np.arange(RP)
    gy = gy0 + np.arange(RH)
    inx, iny = (gx >= 0) & (gx < w), (gy >= 0) & (gy < h)
    raw = np.where(iny[:, None] & inx[None, :], gy[:, None] * w + gx[None, :], -1)
    ry_lo, ry_hi = max(0, -gy0), min(RH, h - gy0)
    if gx0 < 0 or gx0 + need_w > w:                          # column pass, in-image rows
        rx = np.arange(need_w)
        out = (gx0 + rx < 0) | (gx0 + rx >= w)
        m = reflect101(gx0 + rx, w) - gx0
        ok = out & (m >= 0) & (m < RP)
        if ry_hi > ry_lo:
            raw[ry_lo:ry_hi, rx[ok]] = raw[ry_lo:ry_hi, m[ok]]
    if ry_lo > 0 or ry_hi < RH:                              # row pass, whole rows
        rows = [ry for ry in range(RH) if ry < ry_lo or ry >= ry_hi]
        for ry in rows:
            m = int(reflect101([gy0 + ry], h)[0]) - gy0
            if 0 <= m < RH:
                raw[ry, :need_w] = raw[m, :need_w]
    return raw


def check_shifted_kernel(name, w, h):
    """Every output pixel of the kernel's grid over a w x h image is produced exactly once, every box starts on a 16-byte
    boundary, and every cell an output reads (its (2R+1)^2 window, inside the NEED x RH part of the box) holds the
    BORDER_REFLECT_101 pixel."""
    TW, TH, RP, NEED, R = shifted_kernels()[name]
    RH = TH + 2 * R
    tx, ty = tma_tiles_x(w, R), (h + TH - 1) // TH
    covered = np.zeros(w, np.int64)
    for bx in range(tx):
        x0 = bx * TW - (16 - R)
        gx0 = x0 - R
        assert gx0 % 16 == 0, (name, w, bx, gx0)
        xs = np.arange(max(x0, 0), min(x0 + TW, w))
        covered[xs] += 1
        for by in range(ty):
            y0 = by * TH
            gy0 = y0 - R
            ys = np.arange(y0, min(y0 + TH, h))
            if len(xs) == 0 or len(ys) == 0:
                continue
            c_lo, c_hi = xs[0] - R - gx0, xs[-1] + R - gx0          # box columns / rows the outputs read
            r_lo, r_hi = ys[0] - R - gy0, ys[-1] + R - gy0
            assert 0 <= c_lo and c_hi < NEED and 0 <= r_lo and r_hi < RH, (name, w, h, bx, by)
            interior = x0 >= R and x0 - R + NEED <= w and y0 >= R and y0 + TH + R <= h
            if interior:
                continue   # no fix-up; the box is inside the image
            raw = reflect_fix_model(gx0, gy0, w, h, RH, RP, NEED)
            cols = reflect101(gx0 + np.arange(c_lo, c_hi + 1), w)
            rows = reflect101(gy0 + np.arange(r_lo, r_hi + 1), h)
            want = rows[:, None] * w + cols[None, :]
            got = raw[r_lo:r_hi + 1, c_lo:c_hi + 1]
            bad = np.argwhere(got != want)
            assert len(bad) == 0, (name, w, h, bx, by, bad[:4].tolist())
    assert (covered == 1).all(), (name, w, np.flatnonzero(covered != 1)[:8])


def check_fast_kernel(w, h):
    """k_fast_nms: tiles of FN_OW x FN_OH outputs cover every pixel once; the 96 x 38 box from the 16-byte boundary at
    or below x0 - 4 holds the 70 x 38 pixels the scores and the NMS of the tile read."""
    OW, OH = T["FN_OW"], T["FN_OH"]
    tx, ty = (w + OW - 1) // OW, (h + OH - 1) // OH
    covx = np.zeros(w, np.int64)
    covy = np.zeros(h, np.int64)
    for bx in range(tx):
        x0 = bx * OW
        xs = (x0 - 4) & ~15
        assert xs % 16 == 0 and xs <= x0 - 4 and x0 + OW + 3 < xs + 96, (w, bx)
        boxoff = x0 - 4 - xs
        assert boxoff + 70 <= 96 and (boxoff + 3 + 63) // 4 + 2 <= 96 // 4   # pass A's last word and its right neighbour
        covx[x0:min(x0 + OW, w)] += 1
    for by in range(ty):
        y0 = by * OH
        assert (OH + 2) + 6 <= 38   # score rows y0 - 1 .. y0 + OH, ring +-3
        covy[y0:min(y0 + OH, h)] += 1
    assert (covx == 1).all() and (covy == 1).all(), (w, h)


# ---- ORB level sizes -----------------------------------------------------------------------------------------------
def orb_level_sizes(w, h, nlevels=4, scale_factor=1.2):
    """orb_build: level l is cv_round_f(w * (1.0f / (float)pow(scaleFactor, l))) in float arithmetic, half to even."""
    out = []
    for l in range(nlevels):
        sc = np.float32(math.pow(float(np.float32(scale_factor)), l))
        inv = np.float32(1.0) / sc
        out.append((int(np.rint(np.float32(w) * inv)), int(np.rint(np.float32(h) * inv))))
    return out


def orb_min_side(edge=ORB_MIN_EDGE, nlevels=4, scale_factor=1.2):
    """The smallest side every level keeps at >= 2 edge + 8 (ORB accepts it; one less is PLF_ERR_INVALID)."""
    need = 2 * edge + 8
    s = need
    while min(orb_level_sizes(s, s, nlevels, scale_factor)[-1]) < need:
        s += 1
    return s


def orb_ok(w, h, nlevels=4, edge=ORB_MIN_EDGE, scale_factor=1.2):
    need = 2 * edge + 8
    return all(a >= need and b >= need for a, b in orb_level_sizes(w, h, nlevels, scale_factor))


# ---- the sweep -----------------------------------------------------------------------------------------------------
def x_boundaries():
    """{kind: widths}: k T and k T +- 1 of the unshifted tile grids (FAST, the generic LBD blur, the sweep's LSD grid BQ),
    64 k - (16 - R) and +- 1 of the shifted ones (and of the sweep's shifted LSD grid BF at the 5- and 7-tap radii)."""
    out = {}
    for name, t in (("FN_OW", T["FN_OW"]), ("BQ_TW", T["BQ_TW"]), ("LBD_TW", T["LBD_TW"])):
        out[name] = sorted({k * t + d for k in (1, 2) for d in (-1, 0, 1)})
    grids = {name: (TW, R) for name, (TW, _, _, _, R) in shifted_kernels().items()}
    grids.update({f"BF_TW_r{r}": (T["BF_TW"], r) for r in (2, 3)})
    for name, (TW, R) in grids.items():
        out[name] = sorted({TW * k - (16 - R) + d for k in (1, 2, 3) for d in (-1, 0, 1)})
    return out


def y_boundaries():
    out = {}
    for name in ("FN_OH", "OBF_TH", "BF_TH", "BQ_TH", "LSD_PRE_TH", "LBF_TH", "LBD_TH"):
        out[name] = sorted({k * T[name] + d for k in (1, 2, 3) for d in (-1, 0, 1)})
    return out


def sweep_widths():
    ws = sorted({v for vs in x_boundaries().values() for v in vs})
    for r in range(16):                       # every residue mod 16, near a multiple of 16 and a shifted boundary
        if not any(v % 16 == r for v in ws):
            ws.append(192 + r)
    return sorted(ws)


def sweep_heights():
    return sorted({v for vs in y_boundaries().values() for v in vs})


def sweep_shapes():
    """(w, h) pairs: every width of sweep_widths() and every height of sweep_heights() at least once, cycled against
    each other (the largest heights go with the smallest widths, so no image gets large)."""
    ws, hs = sweep_widths(), sweep_heights()[::-1]
    n = max(len(ws), len(hs))
    return [(ws[i % len(ws)], hs[i % len(hs)]) for i in range(n)]


# LSD has no size floor of its own beyond 3 x 3 (plf_lsd rejects smaller images): 1-pixel and 2-pixel sides are refused,
# sizes below the blur radius and below one tile run
LSD_REFUSED = [(1, 1), (1, 9), (9, 1), (2, 2), (2, 30), (30, 2)]
LSD_TINY = [(3, 3), (3, 40), (40, 3), (4, 4), (5, 7), (7, 5), (6, 6), (8, 8), (9, 17), (20, 10), (33, 15)]


def orb_boundary_shapes(nlevels, lo, hi, h_lo=None):
    """ORB base sizes whose level sizes on levels >= 1 (found with ORB's own rounding) hit the FAST and ORB-blur
    boundaries: one width per x boundary and one height per y boundary, paired; every shape is one ORB accepts."""
    xb = sorted(set(x_boundaries()["FN_OW"]) | set(x_boundaries()["orb_blur7"]))
    yb = sorted(set(y_boundaries()["FN_OH"]) | set(y_boundaries()["OBF_TH"]))
    h_lo = h_lo or lo
    ws, hs = [], []
    for b in xb:
        for w in range(lo, hi):
            if b in [s[0] for s in orb_level_sizes(w, w, nlevels)[1:]]:
                ws.append(w)
                break
    for b in yb:
        for h in range(h_lo, hi):
            if b in [s[1] for s in orb_level_sizes(h, h, nlevels)[1:]]:
                hs.append(h)
                break
    ws, hs = sorted(set(ws)), sorted(set(hs))[::-1]
    n = max(len(ws), len(hs))
    shapes = [(ws[i % len(ws)], hs[i % len(hs)]) for i in range(n)]
    return [s for s in shapes if orb_ok(*s, nlevels=nlevels)]


ORB_SHAPES_L4 = orb_boundary_shapes(4, orb_min_side(nlevels=4), 420)
ORB_SHAPES_L8 = orb_boundary_shapes(8, orb_min_side(nlevels=8), 900)


def orb_size_edges():
    """(nlevels, edge, smallest accepted side): the shapes at and one pixel below ORB's minimum, per axis."""
    out = []
    for nl, edge in ((1, ORB_MIN_EDGE), (4, ORB_MIN_EDGE), (8, ORB_MIN_EDGE), (4, 31)):
        out.append((nl, edge, orb_min_side(edge, nl)))
    return out


def kitti_class_shapes():
    """Two full-width shapes (1200..1280 x 360..400) whose pyramids put the most levels on a FAST / ORB-blur boundary."""
    xb = set(x_boundaries()["FN_OW"]) | set(x_boundaries()["orb_blur7"])
    xb |= {b + 64 * k for b in x_boundaries()["orb_blur7"] for k in range(1, 20)}
    xb |= {b + 62 * k for b in x_boundaries()["FN_OW"] for k in range(1, 20)}
    yb = {T["FN_OH"] * k + d for k in range(1, 15) for d in (-1, 0, 1)} | {T["OBF_TH"] * k + d for k in range(1, 15) for d in (-1, 0, 1)}
    hits = lambda w, h: sum((a in xb) + (b in yb) for a, b in orb_level_sizes(w, h, 8)[1:])
    best = sorted(((hits(w, h), w, h) for w in range(1200, 1281) for h in range(360, 401, 3)), reverse=True)
    out = [(best[0][1], best[0][2])]
    out.append(next((w, h) for _, w, h in best if w % 16 != out[0][0] % 16 and h != out[0][1]))
    return out


# ---- the library's resize tables (host code of libplslam_b200.so) --------------------------------------------------
def _plf_lib():
    import plslam_b200 as plf
    return plf.load_library()


def resize_tables(sw, dw):
    """plf_linear_coeffs_host + plf_resize_packed_len + plf_resize_pack_x (C++ host functions of the library) for one
    axis: (ofs, c1, packed int32 [len])."""
    lib = _plf_lib()
    coeffs = lib["_Z22plf_linear_coeffs_hostiidPiS_"]
    coeffs.argtypes = [C.c_int, C.c_int, C.c_double, C.c_void_p, C.c_void_p]
    plen = lib["_Z21plf_resize_packed_leni"]
    plen.restype, plen.argtypes = C.c_size_t, [C.c_int]
    pack = lib["_Z17plf_resize_pack_xPKiS0_iPi"]
    pack.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    ofs, c1 = np.zeros(dw, np.int32), np.zeros(dw, np.int32)
    coeffs(sw, dw, 1.0 / (dw / sw), ofs.ctypes.data, c1.ctypes.data)
    n = int(plen(dw))
    buf = np.full(max(n, 2 * dw) + 64, -7, np.int32)     # slack: a short length must not make this test write past it
    pack(ofs.ctypes.data, c1.ctypes.data, dw, buf.ctypes.data)
    return ofs, c1, buf[:n]


def check_resize_exact4(sw, dw):
    """k_resize_exact4 over a source row of sw bytes: the packed table has whole groups of four columns (it is read with
    two 128-bit loads per group, so a short table would be read past its end), padding entries repeat the last column,
    and every group's byte pairs lie in the 8-byte window from its first column, inside the row."""
    assert sw <= 1.9 * dw
    ofs, c1, packed = resize_tables(sw, dw)
    dw4 = (dw + 3) & ~3
    assert len(packed) == 2 * dw4, (sw, dw, len(packed))
    p = packed.reshape(dw4, 2)
    idx = np.minimum(np.arange(dw4), dw - 1)
    assert np.array_equal(p[:, 0], ofs[idx]), (sw, dw)
    assert np.array_equal(p[:, 1], (256 - c1[idx]) | (c1[idx] << 16)), (sw, dw)
    g = p[:, 0].reshape(-1, 4)
    d = g - g[:, :1]
    assert (d >= 0).all() and (d <= 6).all(), (sw, dw)
    assert ofs.min() >= 0 and (ofs + 1).max() <= max(sw - 1, 1), (sw, dw)


# ============================================================== tests ===============================================
def test_tile_constants_read_from_the_kernels():
    assert T["FN_OW"] < 64 and T["FN_OH"] < 32          # the FAST tile + its 1-pixel NMS halo fits the 64 x 32 score tile
    for name, (TW, TH, RP, NEED, R) in shifted_kernels().items():
        assert TW == 64 and RP % 16 == 0 and NEED <= RP and TW + 2 * R <= NEED, name
    assert T["LSD_PRE_BOXW"] % 16 == 0 and T["LSD_PRE_HW"] + 2 * max(LSD_RADII) <= T["LSD_PRE_BOXW"]
    assert max(LSD_RADII) == T["LSD_PRE_KS_MAX"] // 2


def test_sweep_covers_residues_and_boundaries():
    ws, hs = sweep_widths(), sweep_heights()
    shapes = sweep_shapes()
    assert {w for w, _ in shapes} == set(ws) and {h for _, h in shapes} == set(hs)
    assert {w % 16 for w in ws} == set(range(16))
    assert any(w % 16 == 0 for w in ws) and any(w % 16 for w in ws)
    for name, bs in x_boundaries().items():
        assert set(bs) <= set(ws), name
    for name, bs in y_boundaries().items():
        assert set(bs) <= set(hs), name
    # each tiled kernel at k T, k T +- 1 (unshifted) and 64 k - (16 - R), +- 1 (shifted)
    for t in (T["FN_OW"], T["BQ_TW"], T["LBD_TW"]):
        assert all(k * t + d in ws for k in (1, 2) for d in (-1, 0, 1)), t
    for _, (TW, _, _, _, R) in shifted_kernels().items():
        assert all(TW * k - (16 - R) + d in ws for k in (1, 2, 3) for d in (-1, 0, 1)), R
    for t in (T["FN_OH"], T["OBF_TH"], T["BF_TH"], T["BQ_TH"], T["LSD_PRE_TH"], T["LBF_TH"], T["LBD_TH"]):
        assert all(k * t + d in hs for k in (1, 2, 3) for d in (-1, 0, 1)), t
    assert max(max(s) for s in shapes) <= 320


@pytest.mark.parametrize("nlevels", [4, 8])
def test_orb_sweep_hits_level_boundaries(nlevels):
    """The ORB base sizes put FAST and ORB-blur tile boundaries on levels >= 1, in both axes; all are accepted sizes."""
    shapes = ORB_SHAPES_L4 if nlevels == 4 else ORB_SHAPES_L8
    xb = set(x_boundaries()["FN_OW"]) | set(x_boundaries()["orb_blur7"])
    yb = set(y_boundaries()["FN_OH"]) | set(y_boundaries()["OBF_TH"])
    lv = [orb_level_sizes(w, h, nlevels)[1:] for w, h in shapes]
    hit_x = {a for levels in lv for a, _ in levels} & xb
    hit_y = {b for levels in lv for _, b in levels} & yb
    reachable_x = {b for b in xb if b >= 2 * ORB_MIN_EDGE + 8}
    reachable_y = {b for b in yb if b >= 2 * ORB_MIN_EDGE + 8}
    assert hit_x == reachable_x, sorted(reachable_x - hit_x)
    assert hit_y == reachable_y, sorted(reachable_y - hit_y)
    assert all(orb_ok(w, h, nlevels) for w, h in shapes)
    for w, h in kitti_class_shapes():
        assert orb_ok(w, h, 8) and w >= 1200


def test_orb_minimum_size_model():
    """orb_min_side is the smallest accepted side (top level = 2 edge + 8) and one pixel less leaves some level short."""
    for nl, edge, s in orb_size_edges():
        need = 2 * edge + 8
        assert orb_ok(s, s, nl, edge) and min(orb_level_sizes(s, s, nl)[-1]) in (need, need + 1)
        assert not orb_ok(s - 1, s, nl, edge) and not orb_ok(s, s - 1, nl, edge)
    assert orb_size_edges()[0][2] == 2 * ORB_MIN_EDGE + 8


def all_model_shapes():
    shapes = set(sweep_shapes()) | set(LSD_TINY) | set(ORB_SHAPES_L4) | set(ORB_SHAPES_L8) | set(kitti_class_shapes())
    for nl, edge, s in orb_size_edges():
        shapes |= {(s, s), (s - 1, s), (s, s - 1)}
    return sorted(shapes)


def test_tile_model_every_shape():
    """For every shape of the sweep (and every ORB level of the ORB shapes): the shifted blur grids and the FAST grid
    cover each pixel once, every TMA box starts on a 16-byte boundary, and plf_tma_reflect_fix leaves the reflected pixel
    in every cell an output reads (no mirror it needs lies outside the box)."""
    n = 0
    for w, h in all_model_shapes():
        levels = [(w, h)]
        if orb_ok(w, h, 8):
            levels = orb_level_sizes(w, h, 8)
        elif orb_ok(w, h, 4):
            levels = orb_level_sizes(w, h, 4)
        for lw, lh in levels:
            names = ["orb_blur7"] if orb_ok(lw, lh, 1) else []
            if lw >= 8 and lh >= 8:
                names.append("lbd_blur5_sobel")    # smaller images take the generic LBD kernel (reflect on load)
            for name in names:
                check_shifted_kernel(name, lw, lh)
                n += 1
            if orb_ok(lw, lh, 1):
                check_fast_kernel(lw, lh)
    assert n > 300


def test_reflect_model_detects_a_skipped_column_pass():
    """The model is not vacuous: without the column pass a left-border tile reads zero-filled cells."""
    TW, TH, RP, NEED, R = shifted_kernels()["orb_blur7"]
    RH = TH + 2 * R
    gx0, gy0 = -16, -R
    raw = reflect_fix_model(gx0, gy0, 100, 60, RH, RP, NEED)
    assert raw[R, 16 - 1] == R * 0 + 1 and raw[R, 16 - 3] == 3    # pixel (-1, 0) -> (1, 0), (-3, 0) -> (3, 0)
    gx = gx0 + np.arange(RP)
    plain = np.where((gx >= 0) & (gx < 100), gx, -1)
    assert (plain[16 - R:16] == -1).all()


def test_resize_tables_every_level(built):
    """The resize tables of every ORB level of the ORB shapes and of the LSD resample of every sweep shape (scale 1.2 and
    the param_cases scales), taken from the library's host code."""
    pairs = set()
    for w, h in sorted(set(ORB_SHAPES_L4) | set(ORB_SHAPES_L8) | set(kitti_class_shapes())):
        for nl in (4, 8):
            if orb_ok(w, h, nl):
                lv = orb_level_sizes(w, h, nl)
                pairs |= {(lv[l - 1][0], lv[l][0]) for l in range(1, nl)} | {(lv[l - 1][1], lv[l][1]) for l in range(1, nl)}
    scales = sorted({c.get("lsd_scale", 1.2) for c in [{}, *LSD_CASES.values()]} - {1.0})
    for w, h in sweep_shapes() + LSD_TINY:
        for sc in scales:
            for s in (w, h):
                d = int(np.rint(s * sc))
                if d >= 3 and s <= 1.9 * d:
                    pairs.add((s, d))
    for sw, dw in sorted(pairs):
        check_resize_exact4(sw, dw)
    assert any(dw % 4 for _, dw in pairs) and any(dw % 4 == 0 for _, dw in pairs)


# ---- the LSD pre-grow kernel's boxes (k_lsd_pre, lsd_pre_geom) -------------------------------------------------------
def lsd_tables(s, d, scale):
    """The LSD resample table of one axis as the library builds it (plf_linear_coeffs_host at 1 / scale): ofs."""
    coeffs = _plf_lib()["_Z22plf_linear_coeffs_hostiidPiS_"]
    coeffs.argtypes = [C.c_int, C.c_int, C.c_double, C.c_void_p, C.c_void_p]
    ofs, c1 = np.zeros(d, np.int32), np.zeros(d, np.int32)
    coeffs(s, d, 1.0 / scale, ofs.ctypes.data, c1.ctypes.data)
    return ofs


def lsd_pre_foot(ox, oy, xa, xl, ya, yl, R):
    """lsd_pre_foot: (bxc, sx1, sy0, sy1)"""
    return ((int(ox[xa]) - R) & ~15) + R, int(ox[xl]) + 1, int(oy[ya]), int(oy[yl]) + 1


def lsd_pre_launch(ox, oy, W, H, R):
    """lsd_pre_geom's TH, NP and PW: the most rows and the fewest pieces whose footprints fit the box."""
    th = next(t for t in range(T["LSD_PRE_TH"], 0, -1)
              if all(lsd_pre_foot(ox, oy, 0, 0, y0, min(y0 + t, H - 1), R)[3] - oy[y0] + 1 + 2 * R <= T["LSD_PRE_BOXH"]
                     for y0 in range(0, H, t)))
    seg = T["LSD_SEG"]
    for np_ in range(1, seg + 2):
        pw = ((seg + np_) // np_ + 3) & ~3
        ok = True
        for x0 in range(0, W, seg):
            nsc = min(seg + 1, W - x0)
            for u0 in range(0, nsc, pw):
                bxc, sx1, _, _ = lsd_pre_foot(ox, oy, x0 + u0, x0 + min(u0 + pw, nsc) - 1, 0, 0, R)
                ok = ok and sx1 - bxc + 1 <= T["LSD_PRE_HW"]
        if ok:
            return th, np_, pw
    raise AssertionError("no piece count fits")


def check_lsd_pre(w, h, scale, R):
    """Every piece of every CTA of k_lsd_pre over a w x h image: its box starts on a 16-byte boundary, the blurred columns
    and rows the resample reads (ofs, ofs + 1) and their blur halo lie inside the box, the packed resample's 12-byte read
    lies inside the blurred tile's row, and every cell outside the image among those the blur reads is rebuilt from a
    mirror cell inside the box (so it holds its BORDER_REFLECT_101 pixel).  Returns (TH, NP)."""
    W, H = (w, h) if scale == 1.0 else (int(np.rint(w * scale)), int(np.rint(h * scale)))
    if W < 3 or H < 3:
        return None
    ox, oy = lsd_tables(w, W, scale), lsd_tables(h, H, scale)
    th, np_, pw = lsd_pre_launch(ox, oy, W, H, R)
    BW, BH, seg = T["LSD_PRE_BOXW"], T["LSD_PRE_BOXH"], T["LSD_SEG"]
    for X0 in range(0, W, seg):
        nsc = min(seg + 1, W - X0)
        for Y0 in range(0, H, th):
            nsr = min(th + 1, H - Y0)
            for u0 in range(0, nsc, pw):
                u1 = min(u0 + pw, nsc)
                bxc, sx1, sy0, sy1 = lsd_pre_foot(ox, oy, X0 + u0, X0 + u1 - 1, Y0, min(Y0 + th, H - 1), R)
                gx0, gy0 = bxc - R, sy0 - R
                assert gx0 % 16 == 0, (w, h, scale, X0, u0)
                ncol, nrow = sx1 - bxc + 1, sy1 - sy0 + 1
                need_w, need_h = ncol + 2 * R, nrow + 2 * R
                assert ncol <= T["LSD_PRE_HW"] and need_w <= BW and need_h <= BH, (w, h, scale, X0, Y0, u0)
                cols, rows = ox[X0 + u0:X0 + u1], oy[Y0:Y0 + nsr]
                assert cols.min() >= bxc and cols.max() + 1 <= sx1 and rows.min() >= sy0 and rows.max() + 1 <= sy1
                assert ((cols - bxc) // 4 * 4 + 12 <= BW).all()    # packed form: three words from the aligned word below ofs
                if gx0 >= 0 and gx0 + need_w <= w and gy0 >= 0 and gy0 + need_h <= h:
                    continue
                mx = reflect101(gx0 + np.arange(need_w), w) - gx0
                my = reflect101(gy0 + np.arange(need_h), h) - gy0
                assert mx.min() >= 0 and mx.max() < BW and my.min() >= 0 and my.max() < need_h, (w, h, scale, X0, Y0, u0)
                raw = reflect_fix_model(gx0, gy0, w, h, need_h, BW, need_w)
                want = (gy0 + my)[:, None] * w + (gx0 + mx)[None, :]
                bad = np.argwhere(raw[:, :need_w] != want)
                assert len(bad) == 0, (w, h, scale, X0, Y0, u0, bad[:4].tolist())
    return th, np_


def test_lsd_pre_boxes_every_shape(built):
    """check_lsd_pre for every sweep shape, the tiny LSD sizes and a KITTI-class frame at the default and every LSD case's
    scale and radius (LSD_CASES, test_lsd_pre_gpu's LSD_PRE_CASES); the defaults keep TH 16 and one piece, downsampling takes several."""
    from test_lsd_pre_gpu import LSD_PRE_CASES
    settings = {(c.get("lsd_scale", 1.2), lsd_pre_ks(c) // 2) for c in [{}, *LSD_CASES.values(), *LSD_PRE_CASES.values()]}
    assert (1.2, 3) in settings and (1.0, 0) in settings and max(r for _, r in settings) == T["LSD_PRE_KS_MAX"] // 2
    launches = {}
    for w, h in sorted(set(sweep_shapes()) | set(LSD_TINY) | {(1241, 376), (853, 35)}):
        for scale, R in sorted(settings):
            got = check_lsd_pre(w, h, scale, R)
            if got:
                launches.setdefault((scale, R), set()).add(got)
    assert launches[(1.2, 3)] == {(16, 1)}
    assert max(p for _, p in launches[(0.5, 5)]) > 1 and max(p for _, p in launches[(0.35, 7)]) > 1


# ---- the C restatements against cv2 at the new shapes ----------------------------------------------------------------
def geometry_image(w, h, seed):
    """Seeded noise plus an axis-aligned block whose edges lie on the image border and on the first tile seams."""
    rng = np.random.default_rng(seed)
    img = rng.integers(60, 120, (h, w), dtype=np.uint8)
    x1 = min(w, T["FN_OW"] if w > T["FN_OW"] else max(1, w // 2))
    y1 = min(h, T["OBF_TH"] if h > T["OBF_TH"] else max(1, h // 2))
    img[:y1, :x1] = 200
    if w > 51 and h > 4:
        img[h // 3:, 51:min(w, 51 + 64)] = 20       # the seam of the shifted blur grids (x0 = 64 - 13)
    return img


def scene_image(w, h, seed):
    from oracle import synth
    if w < 24 or h < 24:
        return geometry_image(w, h, seed)
    return synth.scene_pair(w=w, h=h, seed=seed, n_rect=max(8, w * h // 400), n_lines=max(4, w * h // 1500))[0]


LSD_CV2_SHAPES = LSD_REFUSED + LSD_TINY + [s for s in sweep_shapes() if s[0] * s[1] <= 12000][::3]


@pytest.mark.parametrize("case", ["default", "sigma0.4_k5", "sigma0.9_k9"])
def test_lsd_oracle_vs_cv2_at_sweep_shapes(built, case):
    """clib.lsd equals cv2's LSD at the tiny and boundary shapes (the device is compared with clib.lsd there)."""
    pytest.importorskip("cv2")
    from oracle import clib
    from oracle.cvref import lsd_cv2
    prm = {} if case == "default" else LSD_CASES[case]
    kw = dict(scale=prm.get("lsd_scale", 1.2), sigma_scale=prm.get("lsd_sigma_scale", 0.6))
    n = 0
    for i, (w, h) in enumerate(LSD_CV2_SHAPES):
        img = scene_image(w, h, i)
        a, b = clib.lsd(img, **kw), lsd_cv2(img, **kw)
        assert a.shape == b.shape and np.array_equal(a, b), (w, h, case)
        n += len(a)
    assert n > 50


def test_orb_oracle_vs_cv2_at_boundary_shapes(built):
    """clib.orb equals cv2's ORB at the level-boundary shapes, the minimum sizes and a KITTI-class shape."""
    pytest.importorskip("cv2")
    from oracle import clib
    from oracle.cvref import orb_cv2
    cases = [(s, 4, ORB_MIN_EDGE) for s in ORB_SHAPES_L4[::2]] + [(s, 8, ORB_MIN_EDGE) for s in ORB_SHAPES_L8[::3]]
    cases += [((s, s), nl, e) for nl, e, s in orb_size_edges()] + [(kitti_class_shapes()[0], 8, ORB_MIN_EDGE)]
    n = 0
    for i, ((w, h), nl, edge) in enumerate(cases):
        img = scene_image(w, h, 100 + i)
        kp, d = clib.orb(img, 500, nlevels=nl, edge_th=edge)
        rk, rd = orb_cv2(img, nfeatures=500, nlevels=nl, edge_th=edge)
        assert len(kp) == len(rk), (w, h, nl)
        n += len(kp)
        for f in ("x", "y", "size", "angle", "response", "octave"):
            assert np.array_equal(kp[f], rk[f]), (w, h, nl, f)
        assert np.array_equal(d, rd), (w, h, nl)
    assert n > 20 * len(cases)
