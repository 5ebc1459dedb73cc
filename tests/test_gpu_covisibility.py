"""GPU suite: ccm_covisibility (KeyFrame::UpdateConnections' counter and ordered connections for a batch,
ccm_slam_b200/csrc/covis.cu) against the host entry point and the oracle, exactly: on the fixture, on the cfg4 and cfg5 observation
shapes, across the shared-table limit and on a keyframe co-observed with thousands of others (the global-memory path); the
capacity rule, the empty batch, repeatability; and shim/KeyFrameConnections_shim.cpp over the real library."""
import numpy as np
import pytest

from ccm_slam_b200 import api, synth
from oracle import pycv
from tests import test_covisibility as TC
from tests import test_shim_covisibility as TS

pytestmark = pytest.mark.gpu

LIMIT = 1024          # distinct observers a keyframe may have on the shared-memory path (covis.cu)


@pytest.fixture(scope="module", autouse=True)
def device():
    if api.device_count() == 0:
        pytest.skip("no CUDA device")
    api.init(0)


def test_device_reproduces_the_fixture():
    for name, sc, want in TC.fixture_cases():
        TC.same(api.covisibility(sc), want)


@pytest.mark.parametrize("cfg", ["cfg4", "cfg5"])
def test_device_equals_host_and_oracle_on_the_ba_shapes(cfg):
    sc = synth.make_covisibility(synth.make_config(cfg), seed=61, same_id_frac=0.01)
    h = api.covisibility(sc, host=True)
    l0 = api.kernel_launches()
    r = api.covisibility(sc, capacity=int(h["conn_ptr"][-1]))
    n_launch = api.kernel_launches() - l0
    TC.same(r, h)
    assert r["status"].mean() > 0.9 and n_launch in (2, 4)
    sub = np.sort(np.random.default_rng(62).choice(sc["batch"], 400, replace=False)).astype(np.int32)
    TC.same(api.covisibility(sc, batch=sub), pycv.oracle(sc, batch=sub))


@pytest.mark.parametrize("hub", [LIMIT - 1, LIMIT, LIMIT + 1, 5000, 7000])
def test_across_the_shared_table_limit_and_high_degree(hub):
    sc = synth.make_covisibility(seed=63 + hub, K=50, P=3000, max_deg=8, hub=hub, null_frac=0.05, dup_frac=0.02, bad_mp_frac=0.0)
    r = api.covisibility(sc)
    o = pycv.oracle(sc)
    TC.same(r, o)
    TC.same(r, api.covisibility(sc, host=True))
    assert r["conn_ptr"][1] - r["conn_ptr"][0] == hub                      # row 0 is co-observed with every other keyframe
    if hub >= 5000:
        assert (r["conn_w"][:hub] >= 15).sum() < hub                         # sub-threshold entries stay in the counter


def test_capacity_refusal_empty_batch_and_repeatability():
    sc = TC.SCENES["maps"]()
    T = int(pycv.oracle(sc)["conn_ptr"][-1])
    rc, o, total = TC._raw(sc, T - 1, fn="ccm_covisibility")
    assert rc == -1 and total == T and all((o[k] == 7).all() for k in TC.KEYS)
    rc1, o1, _ = TC._raw(sc, T, fn="ccm_covisibility")
    rc2, o2, _ = TC._raw(sc, T, fn="ccm_covisibility")
    assert rc1 == rc2 == 0
    for k in TC.KEYS:
        assert o1[k].tobytes() == o2[k].tobytes(), k
    r = api.covisibility(sc, batch=np.zeros(0, np.int32))
    assert r["conn_ptr"].tolist() == [0]
    bad = dict(sc); bad["obs_kf"] = sc["obs_kf"].copy(); bad["obs_kf"][-1] = len(sc["kf_id"])
    with pytest.raises(api.CCMError, match="batch keyframe"):
        api.covisibility(bad)


def test_shim_over_the_real_library():
    sc = TS.scene(64)
    B = len(sc["batch"])
    lit, _, _ = TS.run(sc, 0)
    s = pycv.StandIn(sc, gpu=True)
    c0 = s.stats()
    s.merge(2)
    assert tuple(s.stats() - c0) == (B, 0, 0)
    got = s.members()
    s.close()
    TS.members_equal(got, lit)
    dbl, _, _ = TS.run(sc, 2)
    TS.members_equal(got, dbl)
