"""The keypoint capacity of the ORB extractor, checked on the CPU oracle.

DistributeOctTree keeps one keypoint per quadtree node.  On a level with quota N whose quadtree starts from nIni root nodes it
ends with at most max(4 * nIni, N + 3) nodes; the argument sits next to the capacity in ccm_slam_b200/csrc/orb.cu, and
ccm_orb_max_keypoints returns the sum over the levels.  Here the bound is computed from the oracle's level tables alone and held
against the oracle's per-level keypoint counts, over quotas, scale factors and frame sizes that reach each of its two terms."""
import numpy as np
import pytest

from ccm_slam_b200.synth_images import make_image, make_noise


def level_bound(oracle, cfg, w, h):
    """(bound per level, quota per level, quadtree roots per level)"""
    npl, _, wh = oracle.orb_tables(cfg, w, h)
    bordered = (wh - 2 * (19 - 3)).astype(np.float32)                      # the quadtree spans the level less 16 px on each side
    n_ini = np.floor((bordered[:, 0] / bordered[:, 1]).astype(np.float64) + 0.5).astype(int)   # std::round of a positive float
    return np.maximum(4 * n_ini, npl + 3), npl, n_ini


SIZES = [(752, 480, 8), (1024, 768, 8), (641, 479, 8), (1280, 240, 8), (221, 221, 8), (1280, 160, 4)]


@pytest.mark.parametrize("nfeatures", [8, 100, 1000, 5000])
@pytest.mark.parametrize("w,h,nlevels", SIZES, ids=["%dx%d-%d" % s for s in SIZES])
def test_keypoints_per_level_within_the_bound(oracle, w, h, nlevels, nfeatures):
    cfg = oracle.orb_cfg(nfeatures=nfeatures, nlevels=nlevels)
    bound, npl, n_ini = level_bound(oracle, cfg, w, h)
    for img in (make_image(2, w, h), make_noise(1, w, h)):
        kps, _ = oracle.orb_extract(img, cfg, max_kp=int(bound.sum()) + 1)
        cnt = np.bincount(kps["octave"], minlength=nlevels)
        assert np.all(cnt <= bound), (cnt, bound)
    # white noise fills every node the first split can make, so where the roots outnumber a quarter of the quota the
    # 4 * nIni term is what holds
    if np.all(4 * n_ini > npl + 3):
        assert np.any(cnt > npl + 3)


@pytest.mark.parametrize("scale_factor,nlevels", [(1.1, 12), (1.5, 5), (2.0, 4)])
def test_bound_at_other_scale_factors(oracle, scale_factor, nlevels):
    w, h = 1024, 768
    for nfeatures in (50, 1000):
        cfg = oracle.orb_cfg(nfeatures=nfeatures, scale_factor=scale_factor, nlevels=nlevels)
        bound, _, _ = level_bound(oracle, cfg, w, h)
        kps, _ = oracle.orb_extract(make_noise(4, w, h, 0.7), cfg, max_kp=int(bound.sum()) + 1)
        assert np.all(np.bincount(kps["octave"], minlength=nlevels) <= bound)


def test_wide_frame_reaches_the_bound(oracle):
    """1280x240 white noise with 8 features: 6 to 9 roots per level (the 16 px border weighs more on small levels), every first
    split full, the bound met exactly"""
    cfg = oracle.orb_cfg(nfeatures=8)
    bound, npl, n_ini = level_bound(oracle, cfg, 1280, 240)
    assert n_ini.tolist() == [6, 6, 6, 7, 7, 8, 8, 9] and int(npl.sum()) == 8
    kps, _ = oracle.orb_extract(make_noise(1, 1280, 240), cfg, max_kp=int(bound.sum()) + 1)
    assert len(kps) == int(bound.sum()) == 228
