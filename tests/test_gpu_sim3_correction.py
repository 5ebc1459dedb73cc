"""GPU suite: ccm_sim3_correction (the Sim3 pass of LoopFinder::CorrectLoop / MapMerger::MergeMaps, ccm_slam_b200/csrc/
sim3_correction.cu) against the host entry point and the oracle, bit for bit with NaN as NaN, in both kinds on the BA shapes; three
launches per call, identical bytes across calls, and refused input that writes nothing."""
import numpy as np
import pytest

from ccm_slam_b200 import api, synth
from oracle import pysc

pytestmark = pytest.mark.gpu

SHAPES = {
    "tiny": lambda: synth.make_config("tiny"),
    "small": lambda: synth.make_config("small"),
    "cfg2": lambda: synth.make_config("cfg2"),
    "cfg4": lambda: synth.make_config("cfg4"),
    "cfg5_tenth": lambda: synth.make_config("cfg5", K=1000, P=100000),
}
OUT = ("entry_Tcw", "entry_centre", "mp_entry", "mp_pos", "normal", "max_dist", "min_dist", "status")
EDGES = dict(K=24, P=3000, window=6, null_frac=0.1, dup_frac=0.1, bad_mp_frac=0.05, tagged_frac=0.05, bad_kf_frac=0.3, all_bad_frac=0.08,
             off_ref_frac=0.3, no_ref_frac=0.03, empty_frac=0.15, null_entry_frac=0.15, unlisted_frac=0.05)


def same(a, b):
    for k in OUT:
        assert np.array_equal(a[k], b[k], equal_nan=True), k


@pytest.fixture(scope="module", autouse=True)
def device():
    if api.device_count() == 0:
        pytest.skip("no CUDA device")
    api.init(0)


@pytest.mark.parametrize("kind", ["loop", "merge"])
@pytest.mark.parametrize("name", list(SHAPES))
def test_device_equals_host_and_oracle(name, kind):
    sc = synth.make_sim3_correction(SHAPES[name](), kind=kind, seed=91, unlisted_frac=0.02, all_bad_frac=0.002, off_ref_frac=0.03)
    l0 = api.kernel_launches()
    r = api.sim3_correction(sc)
    assert api.kernel_launches() == l0 + 3
    same(r, api.sim3_correction(sc, host=True))
    same(r, pysc.oracle(sc))
    assert (r["mp_entry"] >= 0).sum() > 0


def test_edge_scenes_and_identical_bytes():
    for seed, kind in ((92, "loop"), (93, "merge")):
        sc = synth.make_sim3_correction(kind=kind, seed=seed, **EDGES)
        a = api.sim3_correction(sc)
        same(a, pysc.oracle(sc))
        b = api.sim3_correction(sc)
        for k in OUT:
            assert a[k].tobytes() == b[k].tobytes(), k
        assert np.isnan(a["normal"]).any(1).sum() > 10


def test_refused_input_writes_nothing():
    sc = synth.make_sim3_correction(kind="merge", seed=94, K=20, P=500)
    sc["entry_kf"] = sc["entry_kf"].copy(); sc["entry_kf"][4] = sc["entry_kf"][0]
    out = api.sim3_correction_out(len(sc["entry_kf"]), len(sc["mp_skip"]))
    for v in out.values():
        v.fill(7)
    l0 = api.kernel_launches()
    with pytest.raises(api.CCMError, match="entry 4: keyframe row"):
        api.sim3_correction(sc, out=out)
    assert api.kernel_launches() == l0
    for v in out.values():
        assert (v == 7).all()


@pytest.mark.parametrize("kind", ["loop", "merge"])
def test_shim_over_the_real_library_matches_the_reference_loop(kind):
    from tests import test_shim_sim3_correction as S
    for name in (kind, kind + "_edges"):
        sc = synth.make_sim3_correction(**S.SCENES[name])
        sc["kind"] = kind
        l0 = api.kernel_launches()
        S.compare(sc, gpu=True)
        assert api.kernel_launches() == l0 + 3                          # the shim's one call
