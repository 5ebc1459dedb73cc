"""ccm_fuse_neighbours on the H100: device == host entry point == flat oracle (oracle/pyfn.py), identical bytes across calls, and one
launch whatever the number of fuse targets."""
import copy

import numpy as np
import pytest

from ccm_slam_b200 import api
from ccm_slam_b200 import synth_match as sm
from oracle import pyfn

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _device():
    if api.device_count() == 0:
        pytest.skip("no CUDA device")
    api.init(0)


def _all_three(sc):
    d = api.fuse_neighbours(sc)
    h = api.fuse_neighbours(sc, host=True)
    rf, rb = pyfn.oracle(sc)
    assert np.array_equal(d[0], h[0]) and np.array_equal(d[1], h[1])
    assert np.array_equal(d[0], rf) and np.array_equal(d[1], rb)
    return d


@pytest.mark.parametrize("seed", [0, 1])
def test_full_size(seed):
    sc = sm.make_fuse_scene(n_first=20, n_second=5, n=1000, seed=seed)
    assert len(sc["entries"]) == 120
    fwd, bwd, settled = _all_three(sc)
    assert (fwd >= 0).sum() > 1000 and (bwd >= 0).sum() > 1000 and settled > 0


def test_one_target_and_no_points():
    sc = sm.make_fuse_scene(n_first=1, n_second=0, n=1000, seed=2)
    fwd, bwd, _ = _all_three(sc)
    assert fwd.shape == (1, 1000) and (fwd >= 0).any()
    e = copy.deepcopy(sc)
    e["cur_point"][:] = -1
    e["cand"] = np.zeros(0, np.int32)
    fwd, bwd, _ = _all_three(e)
    assert (fwd == -1).all() and bwd.shape == (0,)


def test_identical_bytes_and_launch_count():
    sc = sm.make_fuse_scene(n_first=20, n_second=5, n=1000, seed=3)
    l0 = api.kernel_launches()
    a = api.fuse_neighbours(sc)
    l1 = api.kernel_launches()
    b = api.fuse_neighbours(sc)
    assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes() and a[2] == b[2]
    one = sm.make_fuse_scene(n_first=1, n_second=0, n=1000, seed=3)
    l2 = api.kernel_launches()
    api.fuse_neighbours(one)
    assert l1 - l0 == 1 and api.kernel_launches() - l2 == 1


def test_shim_over_the_library():
    """shim/FuseNeighbours_shim.cpp over the real device entry point against the literal restatement, member for member"""
    from tests.test_shim_fuse_neighbours import run_both, same_members
    sc = sm.make_fuse_scene(n_first=8, n_second=4, n=600, seed=9)
    ref, shim, stats = run_both(sc, gpu=True)
    same_members(ref, shim)
    assert stats[0] == 1 and stats[1] >= 1 and "i" in bytes(ref["log"]).decode()
