"""GPU suite: ccm_new_map_points (LocalMapping::CreateNewMapPoints for a keyframe and all its neighbours in one call,
ccm_slam_b200/csrc/new_points.cu) against the host entry point and the sequential oracle, bit for bit — points, order, best2 and
verdicts: on the fixture, on random 20 x 1000 scenes, at 20 x 2000 (the initialisation budget), with one neighbour and on a keyframe
whose features all carry map points; identical bytes across two calls; a launch count that does not grow with the neighbours; the
capacity rule; and shim/NewMapPoints_shim.cpp over the real library."""
import numpy as np
import pytest

from ccm_slam_b200 import api, synth_match as sm
from oracle import pynp
from tests import test_new_map_points as TN
from tests import test_shim_new_map_points as TS

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def device():
    if api.device_count() == 0:
        pytest.skip("no CUDA device")
    api.init(0)


def same(a, b):
    assert len(a[0]) == len(b[0]) and a[0].tobytes() == b[0].tobytes()
    assert np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])


def test_device_reproduces_the_fixture():
    for name, sc, want in TN.fixture_cases():
        same(api.new_map_points(sc["cur"], sc["neighbours"], want_debug=True), want)


@pytest.mark.parametrize("seed", [11, 12, 13])
def test_device_equals_host_and_oracle_on_random_scenes(seed):
    sc = sm.make_new_points_scene(n_nb=20, n=1000, seed=seed, zero_baseline_nb=seed % 20, no_shared_nb=(seed + 7) % 20)
    d = api.new_map_points(sc["cur"], sc["neighbours"], want_debug=True)
    same(d, api.new_map_points(sc["cur"], sc["neighbours"], want_debug=True, host=True))
    same(d, pynp.oracle(sc["cur"], sc["neighbours"]))
    assert len(d[0]) > 300
    assert api.new_map_points(sc["cur"], sc["neighbours"]).tobytes() == d[0].tobytes()      # without the debug arrays


def test_the_initialisation_budget():
    sc = sm.make_new_points_scene(n_nb=20, n=2000, seed=21)
    d = api.new_map_points(sc["cur"], sc["neighbours"], want_debug=True)
    same(d, pynp.oracle(sc["cur"], sc["neighbours"]))
    assert len(d[0]) > 600


def test_one_neighbour_and_no_free_feature():
    sc = sm.make_new_points_scene(n_nb=1, n=1000, seed=22)
    same(api.new_map_points(sc["cur"], sc["neighbours"], want_debug=True), pynp.oracle(sc["cur"], sc["neighbours"]))
    sc = sm.make_new_points_scene(n_nb=3, n=400, seed=23, all_have_mp=True)
    l0 = api.kernel_launches()
    pts, b2, vd = api.new_map_points(sc["cur"], sc["neighbours"], want_debug=True)
    assert api.kernel_launches() == l0                               # nothing to search: no launch
    assert len(pts) == 0 and (b2 == -1).all() and (vd == 0).all()
    assert len(api.new_map_points(sc["cur"], [])) == 0


def test_two_calls_give_identical_bytes():
    sc = sm.make_new_points_scene(n_nb=20, n=1000, seed=24)
    a = api.new_map_points(sc["cur"], sc["neighbours"], want_debug=True)
    for _ in range(3):
        b = api.new_map_points(sc["cur"], sc["neighbours"], want_debug=True)
        assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b))


def test_the_launch_count_does_not_grow_with_the_neighbours():
    sc = sm.make_new_points_scene(n_nb=20, n=1000, seed=25)
    counts = []
    for k in (1, 20):
        l0 = api.kernel_launches()
        api.new_map_points(sc["cur"], sc["neighbours"][:k])
        counts.append(api.kernel_launches() - l0)
    assert counts == [3, 3]


def test_capacity_short_by_one():
    sc = sm.make_new_points_scene(n_nb=6, n=500, seed=26)
    pts = api.new_map_points(sc["cur"], sc["neighbours"])
    with pytest.raises(api.CCMError, match="capacity %d below the %d points needed" % (len(pts) - 1, len(pts))) as e:
        api.new_map_points(sc["cur"], sc["neighbours"], capacity=len(pts) - 1)
    assert e.value.needed == len(pts)
    assert api.new_map_points(sc["cur"], sc["neighbours"], capacity=len(pts)).tobytes() == pts.tobytes()


def test_invalid_input_names_the_neighbour():
    sc = sm.make_new_points_scene(n_nb=3, n=200, seed=27)
    sc["neighbours"][2]["octave"] = sc["neighbours"][2]["octave"].copy()
    sc["neighbours"][2]["octave"][5] = 8
    with pytest.raises(api.CCMError, match="neighbour 2: octave of feature 5 out of range"):
        api.new_map_points(sc["cur"], sc["neighbours"])


def test_the_shim_over_the_real_library():
    TS.test_the_whole_member(gpu=True)
    TS.test_neighbours_skipped_for_their_baseline(gpu=True)
    TS.test_an_early_return_keeps_the_reference_prefix(3, gpu=True)


def test_the_shim_turns_a_refused_call_into_the_references_exception():
    sc = TS.scene()
    sc["neighbours"][1]["octave"] = sc["neighbours"][1]["octave"].copy()
    sc["neighbours"][1]["octave"][0] = 8
    s = pynp.StandIn(sc["cur"], sc["neighbours"], gpu=True)
    with pytest.raises(RuntimeError, match="the member threw"):
        s.run(1)
    assert len(s.members()["pos"]) == 0
    s.close()


@pytest.mark.parametrize("kind", ["reproj2", "dist_zero"])
def test_hand_built_pairs_reach_the_remaining_verdicts(kind):
    sc = TN.single_pair_scene(kind)
    d = api.new_map_points(sc["cur"], sc["neighbours"], want_debug=True)
    same(d, api.new_map_points(sc["cur"], sc["neighbours"], want_debug=True, host=True))
    assert d[2][0, 0] == TN.V[kind]


def test_a_feature_vector_of_empty_nodes_gives_no_point_and_no_launch():
    sc = TN.empty_nodes_scene()
    l0 = api.kernel_launches()
    pts, b2, vd = api.new_map_points(sc["cur"], sc["neighbours"], want_debug=True)
    assert api.kernel_launches() == l0 and len(pts) == 0 and (b2 == -1).all() and (vd == 0).all()
