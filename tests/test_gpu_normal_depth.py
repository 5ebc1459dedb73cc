"""GPU suite: ccm_normal_depth (MapPoint::UpdateNormalAndDepth for a batch, ccm_slam_b200/csrc/normal_depth.cu) against the oracle,
bit for bit with NaN as NaN, on the observer structure of the BA shapes and on every edge case; and shim/MapPoint_shim.cpp over the
real library: the parked path leaves the members the host path leaves."""
import numpy as np
import pytest

from ccm_slam_b200 import api, synth
from oracle import pynd
from tests import test_shim_optimizer_normals as ONS

pytestmark = pytest.mark.gpu

SHAPES = {
    "tiny": lambda: synth.make_config("tiny"),
    "small": lambda: synth.make_config("small"),
    "cfg2": lambda: synth.make_config("cfg2"),
    "cfg4": lambda: synth.make_config("cfg4"),
    "cfg5_tenth": lambda: synth.make_config("cfg5", K=1000, P=100000),
    "awkward": lambda: synth.make_awkward_ba(),
}
KEYS = ("normal", "max_dist", "min_dist", "status")


def same(a, b):
    for k in KEYS:
        assert np.array_equal(a[k], b[k], equal_nan=True), k


@pytest.fixture(scope="module", autouse=True)
def device():
    if api.device_count() == 0:
        pytest.skip("no CUDA device")
    api.init(0)


@pytest.mark.parametrize("name", list(SHAPES))
def test_device_equals_oracle(name):
    sc = synth.make_normal_depth(SHAPES[name](), seed=61, bad_kf_frac=0.05, all_bad_frac=0.002, on_centre_frac=0.002, off_ref_frac=0.03)
    l0 = api.kernel_launches()
    r = api.normal_depth(sc)
    assert api.kernel_launches() == l0 + 1
    same(r, pynd.oracle(sc))
    assert r["status"].sum() > 0.9 * len(r["status"]) - sc["mp_bad"].sum()


def test_device_edge_cases():
    for seed in (62, 63):
        sc = synth.make_normal_depth(seed=seed, K=10, P=3000, bad_kf_frac=0.3, bad_mp_frac=0.1, all_bad_frac=0.1, on_centre_frac=0.1,
                                     off_ref_frac=0.3)
        r = api.normal_depth(sc)
        same(r, pynd.oracle(sc))
        same(r, api.normal_depth(sc, host=True))
        assert np.isnan(r["normal"]).any(1).sum() > 50 and (r["status"] == 0).sum() > 100
    e = synth.make_normal_depth(seed=64, K=3, P=0)
    assert len(api.normal_depth(e)["status"]) == 0
    bad = synth.make_normal_depth(seed=65, K=5, P=50)
    bad["obs_kf"] = bad["obs_kf"].copy(); bad["obs_kf"][-1] = 7
    with pytest.raises(api.CCMError):
        api.normal_depth(bad)


def test_shim_over_the_real_library():
    sc = synth.make_normal_depth(synth.make_config("small"), seed=66, bad_kf_frac=0.1, all_bad_frac=0.01, on_centre_frac=0.01,
                                 off_ref_frac=0.05, map_order=True)
    s = pynd.StandIn(sc, gpu=True)
    c0 = s.stats()
    parked = s.shim(prepare=True)
    assert tuple(s.stats() - c0) == (int(parked["status"].sum()), 0, 0)
    s.close()
    s = pynd.StandIn(sc, gpu=True)
    host = s.shim(prepare=False)
    same(parked, host)
    same(parked, s.literal())
    same(parked, pynd.oracle(sc))
    s.close()


@pytest.mark.parametrize("which", ONS.IDS)
def test_optimizer_write_backs_over_the_real_library(oracle, which):
    """the five write-back loops of shim/Optimizer_shim.cpp with shim/MapPoint_shim.cpp, over ccm_normal_depth on the device: the members
    per-point host computation gives, and one parked value taken per written point"""
    L = ONS.nd_lib(gpu=True)
    if L is None:
        pytest.skip("oracle/_ref/liboptimizer_nd_shim_gpu.so not available")
    _, sc, fn, args, kw = ONS.write_backs(oracle)[ONS.IDS.index(which)]
    ONS.check(sc, *ONS.run(L, sc, fn, *args, **kw))
