"""ccm_search_and_fuse on the H100: device == host entry point == flat oracle (oracle/pysf.py) at full size, identical bytes across
calls, and one launch whatever the number of corrected keyframes."""
import copy

import numpy as np
import pytest

from ccm_slam_b200 import api
from ccm_slam_b200 import synth_match as sm
from oracle import pysf

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _device():
    if api.device_count() == 0:
        pytest.skip("no CUDA device")
    api.init(0)


def _all_three(sc):
    d = api.search_and_fuse(sc)
    h = api.search_and_fuse(sc, host=True)
    assert np.array_equal(d[0], h[0])   # the results; which pairs each side flags for logf may differ in the last bit of its f64 log
    assert np.array_equal(d[0], pysf.oracle(sc))
    return d


@pytest.mark.parametrize("kind,seed", [("loop", 0), ("merge", 1)])
def test_full_size(kind, seed):
    """the loop shape of the probe: 31 corrected keyframes of 1000 features against about 8000 loop points"""
    sc = sm.make_search_and_fuse_scene(kind, n_kf=31, n=1000, n_loop=8000, seed=seed, boundary=200)
    best, settled = _all_three(sc)
    assert (best >= 0).sum() > 5000 and settled > 0


def test_point_count_not_a_multiple_of_32_and_empty():
    sc = sm.make_search_and_fuse_scene("merge", n_kf=3, n=500, n_loop=1001, seed=2)
    P = len(sc["points"]["skip"])
    assert P % 32 != 0
    best, _ = _all_three(sc)
    assert (best >= 0).any()
    e = copy.deepcopy(sc)
    e["points"]["skip"][:] = 1
    best, _ = _all_three(e)
    assert (best == -1).all()
    l0 = api.kernel_launches()
    best, settled = api.search_and_fuse(dict(sc, kfs=[]))
    assert best.shape == (0, P) and settled == 0 and api.kernel_launches() == l0   # no pairs: no launch


def test_identical_bytes_and_launch_count():
    sc = sm.make_search_and_fuse_scene("loop", n_kf=31, n=1000, n_loop=8000, seed=3)
    l0 = api.kernel_launches()
    a = api.search_and_fuse(sc)
    l1 = api.kernel_launches()
    b = api.search_and_fuse(sc)
    assert a[0].tobytes() == b[0].tobytes() and a[1] == b[1]
    one = dict(sc, kfs=sc["kfs"][:1])
    l2 = api.kernel_launches()
    api.search_and_fuse(one)
    assert l1 - l0 == 1 and api.kernel_launches() - l2 == 1


def test_shim_over_the_library():
    """shim/SearchAndFuse_shim.cpp over the real device entry point against the literal restatement, member for member, at both sites"""
    from tests.test_shim_search_and_fuse import run_both, same_members, scene
    for kind, merge, seed in (("loop", False, 6), ("merge", True, 7)):
        ref, shim, stats = run_both(scene(kind, seed), merge, gpu=True)
        same_members(ref, shim)
        assert stats[0] == 1 and stats[1] > 0
