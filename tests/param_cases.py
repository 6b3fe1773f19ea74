"""The front-end parameter cases the suite runs, in one table (plf_params field names).

REFERENCE_CONFIGS  the front-end keys of the reference's other configuration files, copied as literals (file:line in the
                   pl-slam tree) so that no test needs a reference checkout.  config_euroc.yaml is plf_default_params().
ORB_CASES / LSD_CASES  standalone detector settings; oracle/orb.c and oracle/lsd.c equal cv2 4.13 bit-for-bit at each.
PIPELINE_SWEEPS    one-at-a-time changes of each stereo gate, matcher and pose threshold from a base run.
SWITCH_CASES       has_points / has_lines.
INVARIANT          fields the library reads but that cannot change its output; the tests assert exactly that.
REJECTED           fields with a single supported value; anything else is PLF_ERR_INVALID.
OUT_OF_RANGE       values outside a varied field's supported range; PLF_ERR_INVALID too.

tests/test_param_coverage.py checks that every plf_params field is in one of these places.
"""

# config/config/config_kitti.yaml:11-79.  use_fld_lines: true (:13) selects the FLD line detector, which this library
# does not implement; the case runs with LSD.  inlier_k (:53) and f2f_overlap_th (:32) are read but ignored (INVARIANT).
KITTI = dict(
    has_points=1, has_lines=1, best_lr_matches=1,
    max_dist_epip=0.0, min_disp=1.0, min_ratio_12_p=0.75,
    line_sim_th=0.75, stereo_overlap_th=0.75, f2f_overlap_th=0.75, min_line_length=0.025, line_horiz_th=0.1,
    min_ratio_12_l=0.9, ls_min_disp_ratio=0.7,
    homog_th=1e-7, min_features=10, max_iters=100, max_iters_ref=100, min_error=1e-7, min_error_change=1e-7, inlier_k=1.0,
    matching_strategy=0, matching_s_ws=10, matching_f2f_ws=3,
    orb_nfeatures=800, orb_scale_factor=1.2, orb_nlevels=4, orb_edge_th=19, orb_wta_k=2, orb_score=1, orb_patch_size=31,
    orb_fast_th=20,
    lsd_nfeatures=100, lsd_refine=0, lsd_scale=1.2, lsd_sigma_scale=0.6, lsd_quant=2.0, lsd_ang_th=22.5, lsd_log_eps=1.0,
    lsd_density_th=0.6, lsd_n_bins=1024)

# config/config/config.yaml:67-133
CONFIG = dict(
    has_points=1, has_lines=1, best_lr_matches=1,
    max_dist_epip=1.0, min_disp=1.0, min_ratio_12_p=0.75,
    line_sim_th=0.75, stereo_overlap_th=0.85, f2f_overlap_th=0.85, min_line_length=0.05, line_horiz_th=1.0,
    min_ratio_12_l=0.75, ls_min_disp_ratio=0.7,
    homog_th=1e-7, min_features=10, max_iters=5, max_iters_ref=10, min_error=1e-7, min_error_change=1e-7, inlier_k=4.0,
    matching_strategy=3, matching_s_ws=10, matching_f2f_ws=3,
    orb_nfeatures=1200, orb_scale_factor=1.2, orb_nlevels=1, orb_edge_th=19, orb_wta_k=2, orb_score=1, orb_patch_size=31,
    orb_fast_th=20,
    lsd_nfeatures=300, lsd_refine=0, lsd_scale=1.2, lsd_sigma_scale=0.6, lsd_quant=2.0, lsd_ang_th=22.5, lsd_log_eps=1.0,
    lsd_density_th=0.6, lsd_n_bins=1024)

# config/config/config_fast.yaml:11-77
FAST = dict(
    has_points=1, has_lines=1, best_lr_matches=1,
    max_dist_epip=1.0, min_disp=1.0, min_ratio_12_p=0.75,
    line_sim_th=0.75, stereo_overlap_th=0.85, f2f_overlap_th=0.85, min_line_length=0.05, line_horiz_th=1.0,
    min_ratio_12_l=0.75, ls_min_disp_ratio=0.7,
    homog_th=1e-7, min_features=10, max_iters=5, max_iters_ref=10, min_error=1e-7, min_error_change=1e-7, inlier_k=4.0,
    matching_strategy=3, matching_s_ws=10, matching_f2f_ws=3,
    orb_nfeatures=600, orb_scale_factor=1.2, orb_nlevels=1, orb_edge_th=19, orb_wta_k=2, orb_score=1, orb_patch_size=31,
    orb_fast_th=20,
    lsd_nfeatures=100, lsd_refine=0, lsd_scale=1.2, lsd_sigma_scale=0.6, lsd_quant=2.0, lsd_ang_th=22.5, lsd_log_eps=1.0,
    lsd_density_th=0.6, lsd_n_bins=1024)

# config/config/config_full.yaml:11-78.  The file has no matching_strategy key (it writes `matching_stereo : 0`, :55),
# so the library default 0 (descriptor-only association) applies.
FULL = dict(
    has_points=1, has_lines=1, best_lr_matches=1,
    max_dist_epip=0.0, min_disp=1.0, min_ratio_12_p=0.75,
    line_sim_th=0.75, stereo_overlap_th=0.75, f2f_overlap_th=0.75, min_line_length=0.025, line_horiz_th=1.0,
    min_ratio_12_l=0.75, ls_min_disp_ratio=0.7,
    homog_th=1e-7, min_features=10, max_iters=5, max_iters_ref=10, min_error=1e-7, min_error_change=1e-7, inlier_k=4.0,
    matching_strategy=0, matching_s_ws=10, matching_f2f_ws=3,
    orb_nfeatures=1200, orb_scale_factor=1.2, orb_nlevels=4, orb_edge_th=19, orb_wta_k=2, orb_score=1, orb_patch_size=31,
    orb_fast_th=20,
    lsd_nfeatures=300, lsd_refine=0, lsd_scale=1.2, lsd_sigma_scale=0.6, lsd_quant=2.0, lsd_ang_th=22.5, lsd_log_eps=1.0,
    lsd_density_th=0.6, lsd_n_bins=1024)

REFERENCE_CONFIGS = {"kitti": KITTI, "config": CONFIG, "fast": FAST, "full": FULL}

# cv::ORB::create settings away from the defaults (scale factor 1.2, 4 levels, edge 19, FAST threshold 20)
# (orb_fast_th 127 and above - the other arm of the packed rejection test - is run by tests/test_adversarial_images*.py
# on images built for it: the rendered scenes these cases run on keep 38 to 64 corners at 127 / 128 and none at 200, below
# the 100 that test_orb_param_cases and test_oracle_matches_cv2_param_cases require of every case)
ORB_CASES = {
    "sf1.1_l8": dict(orb_scale_factor=1.1, orb_nlevels=8),
    "sf1.5_l4": dict(orb_scale_factor=1.5, orb_nlevels=4),
    "sf2.0_l3": dict(orb_scale_factor=2.0, orb_nlevels=3),
    "l5": dict(orb_nlevels=5),
    "l6": dict(orb_nlevels=6),
    "l7": dict(orb_nlevels=7),
    "edge25_fast7": dict(orb_edge_th=25, orb_fast_th=7),
    "edge31": dict(orb_edge_th=31),
    "fast40": dict(orb_fast_th=40),
}

# cv::createLineSegmentDetector settings away from the defaults (scale 1.2, sigma_scale 0.6, quant 2, ang_th 22.5,
# 1024 bins).  The Gaussian kernel is 1 + 2 ceil(3.717 sigma), sigma = sigma_scale (/ scale below 1): the cases give
# kernels of 3, 5, 9, 11 and 15 taps besides the default 7.
LSD_CASES = {
    "scale0.35_k15": dict(lsd_scale=0.35),                            # sigma 1.714 -> 15 taps
    "scale0.5_k11": dict(lsd_scale=0.5),                              # sigma 1.2 -> 11 taps
    "scale2.0": dict(lsd_scale=2.0),                                  # upsampling, 7 taps
    "sigma0.25_k3": dict(lsd_sigma_scale=0.25),                       # 3 taps
    "sigma0.4_k5": dict(lsd_sigma_scale=0.4),                         # 5 taps
    "sigma0.9_k9": dict(lsd_sigma_scale=0.9),                         # 9 taps
    # 5 taps whose Q8 centre tap is 256 ([0, 0, 256, 0, 0]): one more than the packed-byte fast blur holds
    "sigma0.28_k5_c256": dict(lsd_sigma_scale=0.28),                  # sigma 0.28
    "scale0.9_sigma0.25_k5_c256": dict(lsd_scale=0.9, lsd_sigma_scale=0.25),   # sigma 0.278, downsampling by 0.9
    "quant1": dict(lsd_quant=1.0),
    "quant4": dict(lsd_quant=4.0),
    "ang15": dict(lsd_ang_th=15.0),
    "ang30": dict(lsd_ang_th=30.0),
    "bins1": dict(lsd_n_bins=1),
    "bins64": dict(lsd_n_bins=64),
}


def lsd_ksize(prm):
    """The Gaussian kernel size LSD uses for prm (0 at lsd_scale 1: no resampling)."""
    import math
    scale, sigma = prm.get("lsd_scale", 1.2), prm.get("lsd_sigma_scale", 0.6)
    if scale == 1.0:
        return 0
    sigma = sigma / scale if scale < 1 else sigma
    return 1 + 2 * math.ceil(sigma * math.sqrt(6 * math.log(10)))


def lsd_pre_ks(prm):
    """The taps LSD's pre-grow kernel blurs with for prm (its template argument): lsd_ksize, or 1 at scale 1 and where the
    Q8 centre tap is 256 (every side tap 0: the blur is a copy)."""
    from oracle import clib
    ks = lsd_ksize(prm)
    if ks == 0:
        return 1
    scale, sigma = prm.get("lsd_scale", 1.2), prm.get("lsd_sigma_scale", 0.6)
    return 1 if clib.gaussian_kernel_q8(ks, sigma / scale if scale < 1 else sigma)[ks // 2] == 256 else ks


# one change at a time through the whole pipeline.  base: the run the change is measured against ({} = the defaults);
# moves: what the change must visibly alter there, so that no case is vacuous - "stereo" = n_stereo_pt / n_stereo_ls,
# "pose" = the GN iteration counts or the pose by more than the parity tolerance.
PIPELINE_SWEEPS = {
    # the stereo gates of k_stereo_points / k_stereo_lines (oracle/frontend.py stereo_points / stereo_lines)
    "min_disp20": dict(base={}, change=dict(min_disp=20.0), moves="stereo"),
    "max_dist_epip0": dict(base={}, change=dict(max_dist_epip=0.0), moves="stereo"),
    "ls_min_disp_ratio0.9": dict(base={}, change=dict(ls_min_disp_ratio=0.9), moves="stereo"),
    "stereo_overlap_th0.5": dict(base={}, change=dict(stereo_overlap_th=0.5), moves="stereo"),
    "line_horiz_th1": dict(base={}, change=dict(line_horiz_th=1.0), moves="stereo"),
    "min_line_length0.05": dict(base={}, change=dict(min_line_length=0.05), moves="stereo"),
    "ratio_p0.75_l0.75": dict(base={}, change=dict(min_ratio_12_p=0.75, min_ratio_12_l=0.75), moves="stereo"),
    "best_lr0": dict(base={}, change=dict(best_lr_matches=0), moves="stereo"),
    # windowed association (matching_strategy 3): window width and the line direction gate
    "s_ws4": dict(base=dict(matching_strategy=3), change=dict(matching_s_ws=4), moves="stereo"),
    "line_sim_th0.99": dict(base=dict(matching_strategy=3), change=dict(line_sim_th=0.99), moves="stereo"),
    # pose refinement: stopping thresholds and the Cauchy weight floor
    "gn_stop1e-3": dict(base={}, change=dict(min_error=1e-3, min_error_change=1e-3), moves="pose"),
    "homog_th1": dict(base={}, change=dict(homog_th=1.0), moves="pose"),
}

SWITCH_CASES = {"points_only": dict(has_lines=0), "lines_only": dict(has_points=0)}

# read by the library, no effect on its output: f2f_overlap_th (stvo-pl's matchF2FLines does not gate on it), inlier_k
# (the outlier gate is a fixed chi2 threshold), lsd_log_eps / lsd_density_th (only used when lines are refined)
INVARIANT = {"f2f_overlap_th": 0.3, "inlier_k": 1.0, "lsd_log_eps": 5.0, "lsd_density_th": 0.95}

# a single supported value; every other value is PLF_ERR_INVALID at the first call that needs the detector
REJECTED = {"orb_wta_k": (2, [3, 4]), "orb_score": (1, [0]), "orb_patch_size": (31, [15]), "lsd_refine": (0, [1, 2])}

# outside the supported range of a field that is otherwise varied: PLF_ERR_INVALID as well.  orb_edge_th below 19 would
# let the 37 x 37 orientation / rBRIEF window cross the level border; lsd_n_bins outside [1, 1024]; lsd_scale 0.3 needs a
# 17-tap Gaussian (at most 15)
OUT_OF_RANGE = {"orb_edge_th": [18, 10, 5], "lsd_n_bins": [0, 1025], "lsd_scale": [0.3]}

# fields varied by a named test elsewhere in the suite (tests/test_param_coverage.py checks that the test exists and
# names the field)
VARIED_ELSEWHERE = {
    "matching_f2f_ws": "test_pipeline_gpu.py::test_pipeline_windowed_matching_fallback",
    "min_pt_matches": "test_pipeline_gpu.py::test_pipeline_windowed_matching_fallback",
    "min_ls_matches": "test_pipeline_gpu.py::test_pipeline_windowed_matching_fallback",
    "min_features": "test_params_gpu.py::test_single_feature_kind_too_few_features",
}


def varied_fields():
    """plf_params fields whose non-default values some case runs."""
    import oracle.frontend as ofe
    out = set(VARIED_ELSEWHERE)
    cases = [*REFERENCE_CONFIGS.values(), *ORB_CASES.values(), *LSD_CASES.values(), *SWITCH_CASES.values()]
    cases += [dict(c["base"], **c["change"]) for c in PIPELINE_SWEEPS.values()]
    for case in cases:
        out |= {k for k, v in case.items() if v != ofe.DEFAULTS[k]}
    return out
