"""Pins the ORB part of the CPU oracle against Python cv2 4.13 (the pinned OpenCV generation, SURVEY.md §8(c')) and
checks the reference's constructor tables (S/ORBextractor.cpp:579-639)."""
import os

import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")

from ccm_slam_b200.synth_images import make_image, make_noise


@pytest.fixture(scope="module")
def img():
    return make_image(0)


def test_constructor_tables(oracle):
    cfg = oracle.orb_cfg()
    npl, umax, wh = oracle.orb_tables(cfg, 752, 480)
    assert npl.tolist() == [217, 181, 151, 126, 105, 87, 73, 60]            # SURVEY §8 a16
    assert umax.tolist() == [15, 15, 15, 15, 14, 14, 14, 13, 13, 12, 11, 10, 9, 8, 6, 3]
    assert wh.tolist() == [[752, 480], [627, 400], [522, 333], [435, 278], [363, 231], [302, 193], [252, 161], [210, 134]]


def test_resize_chain_matches_cv2(oracle, img):
    cur = img
    for (w, h) in [(627, 400), (522, 333), (435, 278), (363, 231), (302, 193), (252, 161), (210, 134)]:
        ref = cv2.resize(cur, (w, h), interpolation=cv2.INTER_LINEAR)
        got = oracle.resize_linear_u8(cur, w, h)
        assert np.array_equal(got, ref)
        cur = ref


@pytest.mark.parametrize("w,h,sf,nl", [(752, 480, 1.1, 12), (752, 480, 1.5, 5), (1024, 768, 2.0, 4), (1024, 768, 1.2, 8), (641, 479, 1.2, 8),
                                       (1280, 240, 1.2, 8), (221, 221, 1.2, 8)])
@pytest.mark.parametrize("frame", ["make_image", "noise"])
def test_pyramid_and_blur_of_other_scales_and_sizes_match_cv2(oracle, w, h, sf, nl, frame):
    """every level of the chained resize and its 7x7 blur, for the scale factors and frame sizes the device tests sweep"""
    _, _, wh = oracle.orb_tables(oracle.orb_cfg(scale_factor=sf, nlevels=nl), w, h)
    cur = make_image(4, w, h) if frame == "make_image" else make_noise(3, w, h, 1.0)
    for l in range(nl):
        w_l, h_l = int(wh[l, 0]), int(wh[l, 1])
        if l:
            ref = cv2.resize(cur, (w_l, h_l), interpolation=cv2.INTER_LINEAR)
            assert np.array_equal(oracle.resize_linear_u8(cur, w_l, h_l), ref), l
            cur = ref
        blur = cv2.GaussianBlur(cur, (7, 7), 2, 2, borderType=cv2.BORDER_REFLECT_101)
        assert np.array_equal(oracle.gaussian_blur7(cur), blur), l


def test_gaussian_blur_matches_cv2(oracle, img):
    for im in (img, cv2.resize(img, (210, 134)), np.zeros((40, 50), np.uint8), np.full((33, 47), 255, np.uint8)):
        ref = cv2.GaussianBlur(im, (7, 7), 2, 2, borderType=cv2.BORDER_REFLECT_101)
        assert np.array_equal(oracle.gaussian_blur7(im), ref)
    # the 2.4.13 tap set differs (sum 257): keep it available, do not claim cv2 parity for it
    assert not np.array_equal(oracle.gaussian_blur7(img, taps2413=True), oracle.gaussian_blur7(img))


@pytest.mark.parametrize("thr", [20, 7])
def test_fast_matches_cv2_including_order_and_scores(oracle, img, thr):
    det = cv2.FastFeatureDetector_create(threshold=thr, nonmaxSuppression=True, type=cv2.FAST_FEATURE_DETECTOR_TYPE_9_16)
    for im in (img, img[16:52, 16:52], img[100:136, 300:336]):
        ref = det.detect(np.ascontiguousarray(im))
        xy, sc = oracle.fast(np.ascontiguousarray(im), thr)
        assert len(ref) == len(xy)
        assert [(int(k.pt[0]), int(k.pt[1])) for k in ref] == [tuple(p) for p in xy.tolist()]
        assert [int(k.response) for k in ref] == sc.tolist()


def test_fast_atan2_bit_identical_to_cv2(oracle):
    rng = np.random.default_rng(0)
    m01 = rng.integers(-60000, 60000, size=5000); m10 = rng.integers(-60000, 60000, size=5000)
    for y, x in zip(m01, m10):
        assert np.float32(oracle.fast_atan2(float(y), float(x))) == np.float32(cv2.fastAtan2(float(y), float(x)))
    assert oracle.fast_atan2(0.0, 0.0) == 0.0


def test_descriptor_matches_cv2_orb_on_given_keypoints(oracle, img):
    """cv2.ORB.compute with provided keypoints (angle kept, nlevels=1) is an independent witness of the steered-BRIEF
    arithmetic on the blurred image."""
    orb = cv2.ORB_create(nfeatures=5000, nlevels=1, edgeThreshold=19, patchSize=31, WTA_K=2, scaleFactor=1.2)
    rng = np.random.default_rng(1)
    kps = []
    for _ in range(300):
        x, y = float(rng.integers(19, 752 - 19)), float(rng.integers(19, 480 - 19))
        ang, m01, m10 = oracle.ic_angle(img, x, y)
        kps.append(cv2.KeyPoint(x, y, 31.0, ang, 1.0, 0))
    kps2, desc = orb.compute(img, kps)
    assert len(kps2) == len(kps)
    blurred = cv2.GaussianBlur(img, (7, 7), 2, 2, borderType=cv2.BORDER_REFLECT_101)
    # cv2.ORB blurs its own bordered pyramid buffer; that image differs from cv2.GaussianBlur(img) by +-1 on a few
    # pixels, so a handful of brightness tests between near-equal pixels flip.  The test therefore bounds the Hamming
    # distance (<= 3 bits per descriptor, < 0.1 % of all bits) instead of demanding equality; bit-exactness of the
    # arithmetic itself is pinned by the independent numpy restatement below.
    import re
    src = open(os.path.join(os.path.dirname(__file__), "..", "oracle", "orb_pattern.h")).read()
    pat = np.array([int(v) for v in re.findall(r"-?\d+", src.split("{")[1])]).reshape(512, 2)
    f = np.float32
    total_bits = 0
    for k, d in zip(kps2, desc):
        got = oracle.orb_descriptor(blurred, k.pt[0], k.pt[1], k.angle)
        hd = int(np.unpackbits(got ^ d).sum())
        assert hd <= 3
        total_bits += hd
        ang = f(k.angle) * f(np.pi / 180.0)
        a, b = f(np.cos(ang)), f(np.sin(ang))
        px, py = pat[:, 0].astype(f), pat[:, 1].astype(f)
        ix = np.rint(f(px * a) - f(py * b)).astype(int); iy = np.rint(f(px * b) + f(py * a)).astype(int)
        v = blurred[int(k.pt[1]) + iy, int(k.pt[0]) + ix].astype(int)
        bits = (v[0::2] < v[1::2]).astype(np.uint8)
        assert np.array_equal(np.packbits(bits.reshape(32, 8)[:, ::-1], axis=1).ravel(), got)
    assert total_bits < 0.001 * 256 * len(kps2)


def test_ic_angle_matches_numpy_moments(oracle, img):
    umax = [15, 15, 15, 15, 14, 14, 14, 13, 13, 12, 11, 10, 9, 8, 6, 3]
    for (x, y) in [(100, 100), (400, 240), (730, 460), (19, 19)]:
        m01 = m10 = 0
        for v in range(-15, 16):
            d = umax[abs(v)]
            for u in range(-d, d + 1):
                p = int(img[y + v, x + u]); m10 += u * p; m01 += v * p
        ang, a, b = oracle.ic_angle(img, float(x), float(y))
        assert (a, b) == (m01, m10)
        assert np.float32(ang) == np.float32(cv2.fastAtan2(float(m01), float(m10)))


def test_extract_end_to_end_invariants(oracle, img):
    kps, desc = oracle.orb_extract(img)
    # DistributeOctTree stops at >= N nodes after a 4-way split, so a level may exceed its quota by up to 3
    assert 900 <= len(kps) <= 1000 + 3 * 8 and desc.shape == (len(kps), 32)
    assert np.all(np.diff(kps["octave"]) >= 0)                       # concatenated level by level
    lvl = kps["octave"]; s = 1.2 ** lvl
    assert np.all(kps["x"] / s >= 19 - 1e-3) and np.all(kps["y"] / s >= 19 - 1e-3)
    cnt = np.bincount(lvl, minlength=8)
    assert np.all(cnt <= np.array([217, 181, 151, 126, 105, 87, 73, 60]) + 3)
    assert np.all((kps["angle"] >= 0) & (kps["angle"] < 360.0 + 1e-3))
    # per-level candidate lists equal per-cell cv2.FAST runs (spot check level 0, first cell row)
    cfg = oracle.orb_cfg()
    cand = oracle.orb_level_candidates(img, cfg, 0)
    det20 = cv2.FastFeatureDetector_create(threshold=20, nonmaxSuppression=True)
    det7 = cv2.FastFeatureDetector_create(threshold=7, nonmaxSuppression=True)
    minB, maxBX, maxBY = 16, 752 - 16, 480 - 16
    wCell = int(np.ceil((maxBX - minB) / int((maxBX - minB) / 30))); hCell = int(np.ceil((maxBY - minB) / int((maxBY - minB) / 30)))
    exp = []
    for i in range(int((maxBY - minB) / 30)):
        iniY = minB + i * hCell; maxY = min(iniY + hCell + 6, maxBY)
        if iniY >= maxBY - 3: continue
        for j in range(int((maxBX - minB) / 30)):
            iniX = minB + j * wCell; maxX = min(iniX + wCell + 6, maxBX)
            if iniX >= maxBX - 6: continue
            roi = np.ascontiguousarray(img[iniY:maxY, iniX:maxX])
            k = det20.detect(roi) or det7.detect(roi)
            exp += [(kp.pt[0] + j * wCell, kp.pt[1] + i * hCell, kp.response) for kp in k]
    assert len(exp) == len(cand)
    assert np.array_equal(np.array(exp, np.float32), cand)
