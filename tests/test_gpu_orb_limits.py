"""The device ORB extractor at its limits, stage by stage against the CPU oracle, exact everywhere.

Every frame is checked at each stage: the keypoints field by field and the descriptors, the FAST candidate list before the quadtree
(ccm_orb_debug_candidates against oracle.orb_level_candidates over all levels), every pyramid level against the chained
oracle.resize_linear_u8, and every blurred level (ccm_orb_debug_blurred) against oracle.gaussian_blur7 with the handle's tap set.

  textured frames      white and smoothed noise with 40 000 - 180 000 candidates, where make_image gives about 7 000
  configuration sweep  quotas 100 - 5000, 1 - 12 levels, scale factors 1.1 - 2.0, both FAST threshold orders, both blur tap sets
  sizes                odd, 1024x768 (more than 1 024 FAST cells), wide frames whose quadtree roots exceed a small quota, the
                       smallest frame a handle accepts; the sizes and calls the library refuses, and extraction after a refusal
  input layout         row-padded images through the C ABI
  handle reuse         one handle across frames whose candidate counts differ by more than 10x, and two handles of different
                       blur tap sets used in turn"""
import ctypes as C

import numpy as np
import pytest

from ccm_slam_b200 import api
from ccm_slam_b200.api import CCMError, _chk, _p, lib
from ccm_slam_b200.frontend import KP_DTYPE, ORBextractor
from ccm_slam_b200.synth_images import make_image, make_noise

pytestmark = pytest.mark.gpu

FIELDS = ("x", "y", "size", "angle", "response", "octave")
CCM_ERR_INVALID = -1


@pytest.fixture(scope="module", autouse=True)
def _dev():
    assert api.device_count() > 0
    api.init(0)


def _extractor(c, w, h):
    """c: keyword arguments of oracle.orb_cfg"""
    return ORBextractor(c.get("nfeatures", 1000), c.get("scale_factor", 1.2), c.get("nlevels", 8), c.get("ini_th", 20), c.get("min_th", 7),
                        w, h, bool(c.get("blur_2413", 0)))


def _candidates(ex, max_out=None):
    n = C.c_int32()
    _chk(lib().ccm_orb_debug_candidates(ex._h, None, None, 0, C.byref(n)))
    m = n.value if max_out is None else max_out
    xys = np.zeros((m, 3), np.float32); level = np.zeros(m, np.int32)
    _chk(lib().ccm_orb_debug_candidates(ex._h, _p(xys), _p(level), m, C.byref(n)))
    return xys, level, n.value


def _blurred(ex, level):
    out = np.empty_like(ex.image_pyramid(level))
    _chk(lib().ccm_orb_debug_blurred(ex._h, level, _p(out)))
    return out


def _check_frame(oracle, ex, img, c):
    """extract img on the device and compare every stage with the oracle; returns (keypoints, descriptors, FAST candidate count)"""
    kps, desc = ex(img)
    cfg = oracle.orb_cfg(**c)
    nl = cfg.nlevels
    rk, rd = oracle.orb_extract(img, cfg, max_kp=ex.max_kp + 1)
    assert len(kps) == len(rk), (len(kps), len(rk))
    for f in FIELDS:
        assert np.array_equal(kps[f], rk[f]), f
    assert np.array_equal(desc, rd)
    assert len(kps) <= ex.max_kp
    want = [oracle.orb_level_candidates(img, cfg, l, max_out=400000) for l in range(nl)]
    xys, level, n = _candidates(ex)
    assert n == sum(len(w) for w in want)
    assert np.array_equal(level, np.repeat(np.arange(nl), [len(w) for w in want]))
    assert np.array_equal(xys, np.concatenate(want))
    _, _, wh = oracle.orb_tables(cfg, img.shape[1], img.shape[0])
    cur = img
    for l in range(nl):
        lv = ex.image_pyramid(l)
        assert lv.shape == (wh[l, 1], wh[l, 0])
        if l:
            cur = oracle.resize_linear_u8(cur, int(wh[l, 0]), int(wh[l, 1]))
        assert np.array_equal(lv, cur), l
        assert np.array_equal(_blurred(ex, l), oracle.gaussian_blur7(cur, bool(c.get("blur_2413", 0)))), l
    return kps, desc, n


# ---- textured frames: 40 000 - 180 000 FAST candidates, every level far above its quota ------------------------------------------
@pytest.mark.parametrize("w,h", [(752, 480), (1024, 768)])
@pytest.mark.parametrize("sigma", [0.0, 0.7, 1.0, 1.5])
def test_textured_frames(oracle, w, h, sigma):
    img = make_noise(7, w, h, sigma)
    ex = _extractor({}, w, h)
    kps, _, ncand = _check_frame(oracle, ex, img, {})
    assert ncand > 40000
    # every level holds far more candidates than its quota, so the quadtree fills every quota
    npl, _, _ = oracle.orb_tables(oracle.orb_cfg(), w, h)
    assert np.all(np.bincount(kps["octave"], minlength=8) >= npl)
    ex.close()


# ---- configuration sweep --------------------------------------------------------------------------------------------------------
CONFIGS = [dict(), dict(nfeatures=500), dict(nfeatures=2000), dict(nlevels=4), dict(scale_factor=1.5, nlevels=5), dict(ini_th=40, min_th=12),
           dict(blur_2413=1), dict(nlevels=1), dict(nlevels=12, scale_factor=1.1), dict(scale_factor=2.0, nlevels=4), dict(nfeatures=100),
           dict(nfeatures=5000), dict(ini_th=10, min_th=3), dict(ini_th=20, min_th=20)]


@pytest.mark.parametrize("frame", ["make_image", "noise"])
@pytest.mark.parametrize("c", CONFIGS, ids=lambda c: "-".join("%s=%s" % kv for kv in c.items()) or "default")
def test_configuration_sweep(oracle, c, frame):
    # level 3 of a 480-row frame at scale 2.0 is 60 rows, less than one FAST cell plus the border: that case runs at 1024x768
    w, h = (1024, 768) if c.get("scale_factor") == 2.0 else (752, 480)
    img = make_image(4, w, h) if frame == "make_image" else make_noise(3, w, h, 1.0)
    ex = _extractor(c, w, h)
    kps, _, ncand = _check_frame(oracle, ex, img, c)
    assert len(kps) > min(c.get("nfeatures", 1000), 400) // 2 and ncand > len(kps)
    ex.close()


# ---- sizes ------------------------------------------------------------------------------------------------------------------------
def _extract_raw(ex, img, max_kp):
    kps = np.full(max(max_kp, 1), 7, KP_DTYPE); desc = np.full((max(max_kp, 1), 32), 7, np.uint8); n = C.c_int32(-1)
    rc = lib().ccm_orb_extract(ex._h, _p(img), img.shape[1], _p(kps), max_kp, C.byref(n), _p(desc))
    return rc, n.value, kps, desc


# (1280, 240): 6 to 9 quadtree roots per level, so a level may keep 24 - 36 keypoints whatever its quota
@pytest.mark.parametrize("w,h,c", [(641, 479, {}), (1024, 768, {}), (1280, 240, {}), (1280, 240, dict(nfeatures=100)), (1280, 240, dict(nfeatures=8))],
                         ids=["641x479", "1024x768", "1280x240", "1280x240-100", "1280x240-8"])
def test_frame_sizes(oracle, w, h, c):
    ex = _extractor(c, w, h)
    for img in (make_image(6, w, h), make_noise(1, w, h)):
        kps, _, _ = _check_frame(oracle, ex, img, c)
    if c.get("nfeatures", 1000) <= 100:
        assert len(kps) > c["nfeatures"] + 96           # the quota plus a fixed allowance does not bound these frames
    # a keypoint buffer one short of the count is refused: the count comes back, nothing is written
    rc, n, k, d = _extract_raw(ex, img, len(kps) - 1)
    assert rc == CCM_ERR_INVALID and n == len(kps)
    assert np.all(k["octave"] == 7) and np.all(d == 7)
    rc, n, k, d = _extract_raw(ex, img, len(kps))
    assert rc == 0 and n == len(kps) and np.array_equal(k["x"], kps["x"])
    ex.close()


def _smallest_square(oracle, c):
    """the smallest square frame every pyramid level of which still holds one 30 px FAST cell inside the border (62 px)"""
    cfg = oracle.orb_cfg(**c)
    return next(s for s in range(40, 1000) if (oracle.orb_tables(cfg, s, s)[2] >= 62).all())


def test_smallest_frame_and_refusals(oracle):
    s = _smallest_square(oracle, {})
    assert s == 221
    for w, h in ((s - 1, s), (s, s - 1)):
        with pytest.raises(CCMError) as e:
            ORBextractor(width=w, height=h)
        assert e.value.code == CCM_ERR_INVALID
    ex = ORBextractor(width=s, height=s)
    for img in (make_image(2, s, s), make_noise(2, s, s)):
        _check_frame(oracle, ex, img, {})
    ex.close()


def test_portrait_frame_is_refused_then_the_library_still_works(oracle):
    # (240 - 32) / (752 - 32) rounds to 0 quadtree roots: the reference would index an empty root list
    ex = ORBextractor(width=240, height=752)
    with pytest.raises(CCMError, match="nIni"):
        ex(make_noise(2, 240, 752))
    flat = np.full((752, 240), 90, np.uint8)
    kps, desc = ex(flat)
    assert len(kps) == 0
    ex.close()
    ex = ORBextractor()
    _check_frame(oracle, ex, make_image(5), {})
    ex.close()


# ---- input layout -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("frame", ["make_image", "noise"])
def test_row_padded_input_equals_contiguous(oracle, frame):
    w, h, pad = 752, 480, 37
    img = make_image(8, w, h) if frame == "make_image" else make_noise(8, w, h, 0.7)
    buf = np.full((h, w + pad), 255, np.uint8)
    buf[:, :w] = img
    ex = ORBextractor()
    kps = np.zeros(ex.max_kp, KP_DTYPE); desc = np.zeros((ex.max_kp, 32), np.uint8); n = C.c_int32()
    _chk(lib().ccm_orb_extract(ex._h, _p(buf), w + pad, _p(kps), ex.max_kp, C.byref(n), _p(desc)))
    assert np.array_equal(ex.image_pyramid(0), img)
    k2, d2, _ = _check_frame(oracle, ex, img, {})    # the contiguous call, itself checked against the oracle
    assert n.value == len(k2) > 500
    for f in FIELDS:
        assert np.array_equal(kps[:n.value][f], k2[f]), f
    assert np.array_equal(desc[:n.value], d2)
    ex.close()


# ---- one handle, many frames ------------------------------------------------------------------------------------------------------
def test_one_handle_across_frames(oracle):
    ex = ORBextractor()
    assert _candidates(ex)[2] == 0                    # before the first extract: an empty list
    flat = np.full((480, 752), 127, np.uint8)
    frames = [make_noise(8), flat, make_image(0), make_noise(9, sigma=1.5), make_image(0)]
    counts = []
    for img in frames:
        kps, _, ncand = _check_frame(oracle, ex, img, {})
        counts.append(ncand)
        if img is flat:
            assert len(kps) == 0 and ncand == 0
    assert counts[0] > 10 * counts[2] > 0
    # a short candidate buffer gets the head of the list and the full count
    full = _candidates(ex)
    head = _candidates(ex, max_out=10)
    assert head[2] == full[2] and np.array_equal(head[0], full[0][:10]) and np.array_equal(head[1], full[1][:10])
    ex.close()


def test_handles_keep_their_own_blur_taps(oracle):
    a = ORBextractor()
    b = ORBextractor(blur_2413=True)                  # created after a: must not change what a computes
    img = make_image(1)
    for ex, c in ((a, {}), (b, dict(blur_2413=1)), (a, {})):
        _check_frame(oracle, ex, img, c)
    a.close(); b.close()
