"""GPU suite: ccm_keyframe_culling (the redundancy test of LocalMapping::KeyFrameCullingV3, ccm_slam_b200/csrc/keyframe_culling.cu)
against the host entry point, bit for bit with n_settled, on the fixture, seeded server-shaped scenes, a 150 x 2000-slot scene and
cascade scenes; one launch per call, identical bytes across calls, refused input that writes nothing, no launch without candidates,
and the shim over the real library against the restatement of the member."""
import numpy as np
import pytest

from ccm_slam_b200 import api, synth
from oracle import pykc

pytestmark = pytest.mark.gpu

OUT = ("cull", "n_mps", "n_red", "n_settled")


@pytest.fixture(scope="module", autouse=True)
def device():
    if api.device_count() == 0:
        pytest.skip("no CUDA device")
    api.init(0)


def check(sc):
    l0 = api.kernel_launches()
    d = api.keyframe_culling(sc)
    assert api.kernel_launches() == l0 + 1
    h = api.keyframe_culling(sc, host=True)
    for k in OUT:
        assert np.array_equal(d[k], h[k]), k
    return d


def test_fixture():
    from tests.test_keyframe_culling import fixture
    for sc, w in fixture():
        d = check(sc)
        for k in ("cull", "n_mps", "n_red"):
            assert np.array_equal(d[k], w[k]), k


@pytest.mark.parametrize("kw", [dict(n_c=20, seed=31), dict(n_c=60, seed=32, n_redundant=4), dict(n_c=150, slots=2000, seed=33, n_redundant=6),
                                dict(n_c=0, seed=34), dict(n_c=30, slots=400, seed=35, obs=(3, 9), bad_kf_frac=0.25, no_ref_frac=0.05)])
def test_device_equals_host(kw):
    sc = synth.make_keyframe_culling_scene(**kw)
    d = check(sc)
    assert d["n_settled"] > 0
    o = pykc.oracle(sc)
    for k in o:
        assert np.array_equal(d[k], o[k]), k


def test_identical_bytes():
    sc = synth.make_keyframe_culling_scene(n_c=60, seed=36)
    a, b = api.keyframe_culling(sc), api.keyframe_culling(sc)
    for k in ("cull", "n_mps", "n_red"):
        assert a[k].tobytes() == b[k].tobytes(), k


def test_refused_input_writes_nothing():
    from tests.test_keyframe_culling import refused_cases
    for sc, msg in refused_cases():
        out = api.keyframe_culling_out(len(sc["cand_kf"]))
        for v in out.values():
            v.fill(7)
        l0 = api.kernel_launches()
        with pytest.raises(api.CCMError, match=msg):
            api.keyframe_culling(sc, out=out)
        assert api.kernel_launches() == l0
        for v in out.values():
            assert (v == 7).all()


def test_no_candidates_no_launch():
    sc = synth.make_keyframe_culling_scene(n_c=5, seed=37, edges=False)
    sc.update(cand_kf=np.zeros(0, np.int32), cand_not_erase=np.zeros(0, np.uint8), slot_ptr=np.zeros(1, np.int64),
              slot_mp=np.zeros(0, np.int32), slot_octave=np.zeros(0, np.int32))
    l0 = api.kernel_launches()
    d = api.keyframe_culling(sc)
    assert api.kernel_launches() == l0 and len(d["cull"]) == 0 and d["n_settled"] == 0


@pytest.mark.parametrize("name", ["server20", "edges", "cascades_only"])
def test_shim_over_the_real_library_matches_the_restatement(name):
    from tests import test_shim_keyframe_culling as S
    l0 = api.kernel_launches()
    S.compare(name, gpu=True)
    assert api.kernel_launches() == l0 + 1                        # the shim's one call
