"""Images built to reach what rendered scenes and uniform noise cannot: the internal capacities of the extraction kernels,
floods of equal FAST scores, saturated arithmetic, the extreme entries of the LSD gradient tables and both arms of FAST's packed
rejection test.  Pure numpy, seeded; every generator returns (uint8 image, record) where the record names the generator,
its arguments and what the image is built to provoke.  tests/test_adversarial_images.py measures, with the CPU oracle,
that each image does what its record says.

W x H is the common size of the small cases: 5 x 7 FAST tiles (62 x 30 outputs) on level 0, four pyramid levels above
the smallest ORB accepts, and one context per parameter set serves every image."""
import numpy as np

W, H = 256, 192
FAST_TILE = (62, 30)       # outputs of one k_fast_nms tile
SEAM_W, SEAM_H = 768, 448  # wide and high enough for a lattice of pitch (11, 13) to meet every column and row phase of a tile
ORB_SORT_CAP = 4096        # csrc/orb.cu: survivors of one pyramid level that k_select_sort can order
KL_SORT_CAP = 4096         # csrc/lsd.cu: lines k_keylines can rank when lsd_nfeatures != 0
CAND_CAP_MAX = 32768       # csrc/orb.cu: FAST candidates of one level, min(w h / 9 + 64, 32768)


def cand_cap(w, h):
    return min(w * h // 9 + 64, CAND_CAP_MAX)


def _rec(name, provokes, **args):
    return dict(name=name, args=args, provokes=provokes)


def flat(v, w=W, h=H):
    return np.full((h, w), v, np.uint8), _rec("flat", "saturated input, no corner and no gradient", v=v)


def step_edges(orientation, w=W, h=H):
    """0 / 255 half planes: 'h' (upper half dark), 'v' (left half dark), 'd' (below the diagonal dark)."""
    yy, xx = np.mgrid[0:h, 0:w]
    m = {"h": yy >= h // 2, "v": xx >= w // 2, "d": xx * h >= yy * w}[orientation]
    return (m * 255).astype(np.uint8), _rec("step_edges", "saturated blurs; one maximal edge, |g| = 510 at scale 1",
                                            orientation=orientation)


def blobs(pitch, size, w=W, h=H):
    """Binary image of size x size white squares every `pitch` pixels: every corner of every square scores 254."""
    yy, xx = np.mgrid[0:h, 0:w]
    m = (yy % pitch < size) & (xx % pitch < size)
    return (m * 255).astype(np.uint8), _rec("blobs", "tie flood: every corner has the same FAST score", pitch=pitch, size=size)


def dot_lattice(px, py, phase=(0, 0), w=W, h=H, fg=255, bg=0):
    """Isolated pixels of value fg on bg, every px columns and py rows from `phase`: each is a strict 3 x 3 maximum with a
    full ring.  Pitches coprime to the FAST tile put a corner at every phase of every tile seam."""
    img = np.full((h, w), bg, np.uint8)
    img[phase[1] % py::py, phase[0] % px::px] = fg
    return img, _rec("dot_lattice", "equal-score corners at every tile-seam phase; candidate count", px=px, py=py, phase=phase)


def stripes(period, orientation, w=W, h=H):
    """0 / 255 stripes of `period` pixels each: orientation 'h' varies along y, 'v' along x."""
    yy, xx = np.mgrid[0:h, 0:w]
    m = ((yy if orientation == "h" else xx) // period) % 2 == 1
    return (m * 255).astype(np.uint8), _rec("stripes", "gradients (+-510, 0) / (0, +-510) in every row or column",
                                            period=period, orientation=orientation)


def checker(cell, w=W, h=H):
    """0 / 255 checkerboard with square cells: at scale 1 the 2 x 2 gradient takes the extreme values the tables hold
    (|gx| + |gy| = 510)."""
    yy, xx = np.mgrid[0:h, 0:w]
    m = ((yy // cell) + (xx // cell)) % 2 == 1
    return (m * 255).astype(np.uint8), _rec("checker", "extreme (gx, gy) pairs of the LSD tables", cell=cell)


def _ramp_bg(th, w, h):
    # columns of 0 .. span in runs of five pixels, so that a ring crosses the steps and its differences straddle th
    span = max(0, min(6, 254 - th))
    return np.tile(((np.arange(w) // 5) % (span + 1)).astype(np.int32), (h, 1))


def ramp(th, w=W, h=H):
    """The background of ramp_lattice alone: steps of one grey level, no corner above a threshold of 1."""
    return _ramp_bg(th, w, h).astype(np.uint8), _rec("ramp", "one-level steps: differences of 1 everywhere", th=th)


def ramp_lattice(th, w=W, h=H):
    """Pixels th and th + 1 above a stepped background, every 7 columns and rows (7 is coprime to 62 and 30): ring
    differences of exactly th (no corner) and th + 1 (corner of score th) at orb_fast_th = th."""
    img = _ramp_bg(th, w, h)
    ys, xs = np.mgrid[3:h:7, 3:w:7]
    img[ys, xs] += th + ((ys // 7 + xs // 7) % 2)
    return np.minimum(img, 255).astype(np.uint8), _rec("ramp_lattice", "ring differences of exactly th and th + 1", th=th)


def noise_dense(w=W, h=H, seed=0):
    """Two-level noise (dark 0..39, bright 215..255): as many FAST corners per pixel as noise gives."""
    rng = np.random.default_rng(seed)
    img = np.where(rng.random((h, w)) < 0.5, rng.integers(0, 40, (h, w)), rng.integers(215, 256, (h, w)))
    return img.astype(np.uint8), _rec("noise_dense", "candidate count per level against cand_cap", seed=seed)


def small_cases(th=20):
    """Every generator at the common size, as [(id, image, record)]; the threshold images are built around th."""
    out = [flat(0), flat(255)]
    out += [step_edges(o) for o in "hvd"]
    out += [blobs(8, 3), blobs(11, 5)]
    out += [dot_lattice(4, 4), dot_lattice(7, 7, (3, 5)), dot_lattice(11, 13, (1, 2)), dot_lattice(31, 7),
            dot_lattice(7, 7, fg=0, bg=255)]
    out += [stripes(p, o) for p in (1, 2, 5) for o in "hv"]
    out += [checker(c) for c in (1, 2, 3, 16)]
    out += [ramp(th), ramp_lattice(th), noise_dense()]
    ids = []
    for _, r in out:
        ids.append(r["name"] + "".join(f"_{v}" for v in r["args"].values()).replace(" ", "").replace("(", "").replace(")", "").replace(",", "x"))
    return [(i, img, r) for i, (img, r) in zip(ids, out)]


# ---- plain models of what the kernels form from an image ----------------------------------------------------------
def gradients(img):
    """LSD's 2 x 2 gradient (gx, gy) at every pixel but the last row / column."""
    a = img.astype(np.int32)
    A, B, C, D = a[:-1, :-1], a[:-1, 1:], a[1:, :-1], a[1:, 1:]
    return (D - A) + (B - C), (D - A) - (B - C)


def lsd_index_bounds(img, n_bins=1024, quant=2.0, ang_th=22.5):
    """The largest values the LSD kernels would form on `img` (already at LSD's working scale): the table index
    li = (gx + 510) 1021 + gy + 510, the packed seed entry's gx^2 + gy^2 and column fields, and the magnitude bin."""
    gx, gy = gradients(img)
    li = (gx + 510) * 1021 + gy + 510
    m2 = gx * gx + gy * gy
    rho = quant / np.sin(np.pi * ang_th / 180.0)
    defined = np.sqrt(m2 / 4.0) > rho
    out = dict(li_min=int(li.min()), li_max=int(li.max()), m2_max=int(m2.max()), col_max=511, bin_max=0,
               n_defined=int(defined.sum()))
    if defined.any():
        max_grad = np.sqrt(float(m2[defined].max()) / 4.0)
        out["bin_max"] = int((np.sqrt(m2[defined] / 4.0) * ((n_bins - 1) / max_grad)).astype(np.int64).max())
    return out


def ring_differences(img):
    """centre - ring pixel for the 16 pixels of the FAST ring, at every pixel at least 3 from the border: [16, h-6, w-6]."""
    a = img.astype(np.int32)
    h, w = a.shape
    ring = [(0, 3), (1, 3), (2, 2), (3, 1), (3, 0), (3, -1), (2, -2), (1, -3), (0, -3), (-1, -3), (-2, -2), (-3, -1),
            (-3, 0), (-3, 1), (-2, 2), (-1, 3)]
    c = a[3:h - 3, 3:w - 3]
    return np.stack([c - a[3 + dy:h - 3 + dy, 3 + dx:w - 3 + dx] for dx, dy in ring])
