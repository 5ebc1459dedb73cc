"""CPU suite: shim/ORBextractor_shim.cpp as a drop-in for cslam::ORBextractor.

The shim is compiled against the reference's own cslam/ORBextractor.h and driven through the class interface (constructor, operator(),
getters, the public mvImagePyramid; oracle/ref_extractor_shim_wrap.cpp -> oracle/_ref/libextractor_shim.so) with the device extractor
doubled by the CPU oracle (oracle/ccm_orb_double.cpp).  Its output is compared with the REFERENCE'S OWN ORBextractor.cpp run on the same
image (oracle/_ref/orb_ref_cli): keypoints field by field, descriptors, and the scale tables the class hands to Frame / KeyFrame.
Skipped where the reference tree is absent."""
import ctypes as C
import os

import numpy as np
import pytest

from ccm_slam_b200.synth_images import make_image, make_noise

SO = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "oracle", "_ref", "libextractor_shim.so")


@pytest.fixture(scope="module")
def xlib(oracle):
    if oracle.build_ref() is None or not os.path.exists(SO) or oracle.ref_orb_cli() is None:
        pytest.skip("oracle/_ref/libextractor_shim.so / orb_ref_cli not available")
    return C.CDLL(SO)


def _max_keypoints(xlib, cfg, w, h):
    """ccm_orb_max_keypoints of the library the shim links against"""
    handle = C.c_void_p(); cap = C.c_int32()
    assert xlib.ccm_orb_create(C.byref(cfg), w, h, C.byref(handle)) == 0
    try:
        assert xlib.ccm_orb_max_keypoints(handle, C.byref(cap)) == 0
    finally:
        xlib.ccm_orb_destroy(handle)
    return cap.value


# (1280, 240, 8 features): each level's quadtree starts from 6 to 9 roots and its first split can leave four keypoints per
# root whatever the quota; white noise gives 228 keypoints there
@pytest.mark.parametrize("seed,w,h,nfeat,nlev,sf", [(0, 752, 480, 1000, 8, 1.2), (3, 376, 240, 500, 6, 1.2), (5, 640, 480, 1500, 8, 1.3),
                                                    ("noise", 1280, 240, 8, 8, 1.2)])
def test_extractor_shim_matches_reference_class(xlib, oracle, seed, w, h, nfeat, nlev, sf):
    img = make_noise(1, w, h) if seed == "noise" else make_image(seed, w, h)
    cfg = oracle.orb_cfg(nfeatures=nfeat, nlevels=nlev, scale_factor=sf, blur_2413=1)      # the stand-in reports OpenCV 2.x: the 2.4.13 blur taps
    cap = _max_keypoints(xlib, cfg, w, h)
    kps = np.zeros(cap, oracle.KP_DTYPE); desc = np.zeros((cap, 32), np.uint8); tables = np.zeros((nlev, 4), np.float32)
    pyr = np.zeros(w * h * 4, np.uint8); wh = np.zeros((nlev, 2), np.int32); get = np.zeros(2, np.int32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    n = xlib.xshim_extract(p(np.ascontiguousarray(img)), w, h, nfeat, C.c_float(sf), nlev, 20, 7, p(kps), cap, p(desc), p(tables), p(pyr), p(wh), p(get))
    assert n > 100 and get[0] == nlev and get[1] == n
    rk, rd = oracle.ref_orb_extract(img, cfg)
    assert n == len(rk)
    for f in ("x", "y", "size", "angle", "response", "octave"):
        assert np.array_equal(kps[:n][f], rk[f]), f
    assert np.array_equal(desc[:n], rd)
    # the scale tables of the constructor (S/ORBextractor.cpp:584-600), float arithmetic
    s = np.empty(nlev, np.float32); s[0] = 1
    for i in range(1, nlev):
        s[i] = np.float32(s[i - 1] * np.float32(sf))
    s2 = (s * s).astype(np.float32)
    assert np.array_equal(tables[:, 0], s) and np.array_equal(tables[:, 2], s2)
    assert np.array_equal(tables[:, 1], (np.float32(1) / s).astype(np.float32)) and np.array_equal(tables[:, 3], (np.float32(1) / s2).astype(np.float32))
    # mvImagePyramid: level 0 is the image, level sizes follow cvRound(size * inverse scale)
    assert tuple(wh[0]) == (w, h) and np.array_equal(pyr[:w * h].reshape(h, w), img)
    for l in range(1, nlev):
        assert tuple(wh[l]) == (int(np.rint(np.float32(w) * tables[l, 1])), int(np.rint(np.float32(h) * tables[l, 1])))
