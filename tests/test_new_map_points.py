"""ccm_new_map_points_host (LocalMapping::CreateNewMapPoints for a keyframe and all its neighbours in one call) against the
sequential oracle and independent witnesses, without a GPU.

The oracle (oracle/new_points_oracle.cpp) runs the reference's loop: per neighbour the reference-pinned orc_match_triangulation, the
gates as the reference writes them, has_mp1 set after each accepted point.  The host entry point runs the library's three passes
(candidates per (neighbour, feature), triangulation per pair, first-accepted-neighbour claims).  They must agree bit for bit.
cv::SVD::compute has no single bit pattern in the reference, so the points are also compared with numpy.linalg.svd in f64 and
cv2.SVDecomp in f32 to a tolerance derived from the conditioning of each A."""
import hashlib
import os

import numpy as np
import pytest

from ccm_slam_b200 import api, synth_match as sm
from oracle import pynp, pyoracle

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "new_map_points.npz")
FIXTURE_SCENES = dict(small=dict(n_nb=4, n=60, seed=41, n_nodes=6, zero_baseline_nb=3),
                      big=dict(n_nb=20, n=1000, seed=42, zero_baseline_nb=5, no_shared_nb=7))
VIEW_KEYS = ("desc", "has_mp", "kp_xy", "octave", "angle", "node", "intr", "Tcw", "Ow", "level_sigma2", "scale_factors", "scale_factor")
V = {name: i for i, name in enumerate(api.NEWPTS_VERDICTS)}
MARGIN = 1e-3          # a witness gate value this close (relatively) to its threshold may fall either way
NEAR_FRACTION = 0.005  # of the pairs of a scene


def scene_digest(sc):
    h = hashlib.sha256()
    for i, v in enumerate([sc["cur"]] + sc["neighbours"]):
        for k in VIEW_KEYS + (("F12", "ex", "ey") if i else ()):
            h.update(np.ascontiguousarray(v[k]).tobytes())
    return h.digest()


def fixture_cases():
    g = np.load(GOLDEN)
    for name, kw in FIXTURE_SCENES.items():
        if name == "small":
            views = []
            for i in range(kw["n_nb"] + 1):
                views.append({k: g["small_v%d_%s" % (i, k)] for k in VIEW_KEYS + (("F12", "ex", "ey") if i else ())})
            sc = dict(cur=views[0], neighbours=views[1:])
        else:
            sc = sm.make_new_points_scene(**kw)
            assert scene_digest(sc) == g[name + "_digest"].tobytes(), "the scene generator no longer reproduces the fixture's inputs"
        yield name, sc, (g[name + "_points"], g[name + "_best2"], g[name + "_verdict"])


def same(a, b):
    assert len(a[0]) == len(b[0]) and a[0].tobytes() == b[0].tobytes()
    assert np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])


def host(sc, **kw):
    return api.new_map_points(sc["cur"], sc["neighbours"], want_debug=True, host=True, **kw)


# ---- the f64 witness: the same pairs, everything in double, numpy's SVD -----------------------------------------------------------
def witness_pair(c, v, i, j, svd=None):
    """-> (verdict, X, slack, cond): slack = the smallest relative distance of an evaluated gate value to its threshold; cond = the
    amplification of a perturbation of A into x3D"""
    d = np.float64
    fx1, fy1, cx1, cy1 = (d(x) for x in c["intr"]); fx2, fy2, cx2, cy2 = (d(x) for x in v["intr"])
    T1, T2 = c["Tcw"].astype(d), v["Tcw"].astype(d)
    k1, k2 = c["kp_xy"][i].astype(d), v["kp_xy"][j].astype(d)
    xn1 = np.array([(k1[0] - cx1) / fx1, (k1[1] - cy1) / fy1, 1.0]); xn2 = np.array([(k2[0] - cx2) / fx2, (k2[1] - cy2) / fy2, 1.0])
    r1, r2 = T1[:, :3].T @ xn1, T2[:, :3].T @ xn2
    cosp = r1 @ r2 / (np.linalg.norm(r1) * np.linalg.norm(r2))
    slack = [abs(cosp - 0.9998) / 0.9998]
    if not (0 < cosp < 0.9998):
        return V["parallax"], None, min(slack), None
    A = np.stack([xn1[0] * T1[2] - T1[0], xn1[1] * T1[2] - T1[1], xn2[0] * T2[2] - T2[0], xn2[1] * T2[2] - T2[1]])
    _, s, vt = (svd or np.linalg.svd)(A)
    h = vt[3].astype(d)
    if h[3] == 0:
        return V["w_zero"], None, 0.0, None
    X = h[:3] / h[3]
    cond = s[0] / max(s[2] - s[3], 1e-300) / abs(h[3]) * np.linalg.norm(h)
    for T, name in ((T1, "depth1"), (T2, "depth2")):
        z = T[2, :3] @ X + T[2, 3]
        slack.append(abs(z) / max(np.linalg.norm(X), 1.0))
        if z <= 0:
            return V[name], X, min(slack), cond
    for T, k, intr, s2, name in ((T1, k1, (fx1, fy1, cx1, cy1), d(c["level_sigma2"][c["octave"][i]]), "reproj1"),
                                 (T2, k2, (fx2, fy2, cx2, cy2), d(v["level_sigma2"][v["octave"][j]]), "reproj2")):
        p = T[:, :3] @ X + T[:, 3]
        e = (intr[0] * p[0] / p[2] + intr[2] - k[0]) ** 2 + (intr[1] * p[1] / p[2] + intr[3] - k[1]) ** 2
        slack.append(abs(e - 5.991 * s2) / (5.991 * s2))
        if e > 5.991 * s2:
            return V[name], X, min(slack), cond
    d1, d2 = np.linalg.norm(X - c["Ow"].astype(d)), np.linalg.norm(X - v["Ow"].astype(d))
    if d1 == 0 or d2 == 0:
        return V["dist_zero"], X, 0.0, cond
    rd, ro, rf = d2 / d1, d(c["scale_factors"][c["octave"][i]]) / d(v["scale_factors"][v["octave"][j]]), 1.5 * d(c["scale_factor"])
    slack += [abs(rd * rf - ro) / ro, abs(rd - ro * rf) / (ro * rf)]
    if rd * rf < ro or rd > ro * rf:
        return V["scale"], X, min(slack), cond
    return V["accepted"], X, min(slack), cond


def witness_check(sc, pts, b2, vd, svd=None, eps=np.finfo(np.float32).eps):
    """every pair the library formed against the witness -> (wrong, near a threshold, pairs).  An accepted point must lie within
    32 * eps32 * cond of the witness's; a verdict may differ only where a witness gate value lies within MARGIN of its threshold, or
    where the conditioning says f32 cannot place the point to within MARGIN."""
    at = {(int(p["nb"]), int(p["idx1"])): p for p in pts}
    wrong = near = pairs = 0
    for b, v in enumerate(sc["neighbours"]):
        for i in np.flatnonzero(b2[b] >= 0):
            pairs += 1
            wv, X, slack, cond = witness_pair(sc["cur"], v, int(i), int(b2[b, i]), svd)
            if wv != vd[b, i]:
                if slack < MARGIN or (cond is not None and 32 * eps * cond > MARGIN):
                    near += 1
                else:
                    wrong += 1
                continue
            if wv == V["accepted"]:
                got = at[(b, int(i))]["x3D"].astype(np.float64)
                if not np.linalg.norm(got - X) <= 32 * eps * cond * max(np.linalg.norm(X), 1.0):
                    wrong += 1
    return wrong, near, pairs


def cv2_svd(A):
    import cv2
    w, u, vt = cv2.SVDecomp(A.astype(np.float32), flags=cv2.SVD_FULL_UV)
    return u, w.ravel().astype(np.float64), vt


# ---- tests ------------------------------------------------------------------------------------------------------------------------
def test_oracle_and_host_reproduce_the_fixture():
    for name, sc, want in fixture_cases():
        same(pynp.oracle(sc["cur"], sc["neighbours"]), want)
        same(host(sc), want)


@pytest.mark.parametrize("seed", range(8))
def test_host_equals_oracle_on_random_scenes(seed):
    n_nb = (20, 20, 7, 1, 20, 3, 12, 20)[seed]
    sc = sm.make_new_points_scene(n_nb=n_nb, n=(1000, 400)[seed % 2], seed=100 + seed, zero_baseline_nb=seed % n_nb,
                                  no_shared_nb=(seed + 2) % n_nb if n_nb > 2 else None)
    same(host(sc), pynp.oracle(sc["cur"], sc["neighbours"]))


def test_best2_is_search_for_triangulation_per_neighbour_with_earlier_claims_folded_in():
    sc = sm.make_new_points_scene(n_nb=8, n=600, seed=51)
    pts, b2, vd = host(sc)
    has = sc["cur"]["has_mp"].copy()
    view = lambda v, h: dict(desc=v["desc"], has_mp=h, kp_xy=v["kp_xy"], octave=v["octave"], angle=v["angle"],  # noqa: E731
                             fv=pyoracle.FeatureVector(v["node"]), intr=v["intr"])
    for b, v in enumerate(sc["neighbours"]):
        pairs = pyoracle.match_triangulation(view(sc["cur"], has), view(v, v["has_mp"]), v["F12"], v["ex"], v["ey"], v["level_sigma2"],
                                             v["scale_factors"], False)
        want = np.full(len(has), -1, np.int32); want[pairs[:, 0]] = pairs[:, 1]
        assert np.array_equal(b2[b], want)
        has[pts["idx1"][pts["nb"] == b]] = 1


@pytest.mark.parametrize("witness", ["numpy_f64", "cv2_f32"])
def test_points_and_verdicts_agree_with_an_independent_svd(witness):
    svd, eps = (None, np.finfo(np.float32).eps) if witness == "numpy_f64" else (cv2_svd, 4 * np.finfo(np.float32).eps)
    for name, sc, want in fixture_cases():
        wrong, near, pairs = witness_check(sc, *want, svd=svd, eps=eps)
        print("%s / %s: %d pairs, %d near a threshold, %d wrong" % (name, witness, pairs, near, wrong))
        assert wrong == 0 and near <= max(1, NEAR_FRACTION * pairs)


def test_the_stated_svd_finds_the_null_vector():
    rng = np.random.default_rng(7)
    for _ in range(200):
        A = rng.normal(size=(4, 4)).astype(np.float32)
        x = pynp.svd4_null(A).astype(np.float64)
        _, s, vt = np.linalg.svd(A.astype(np.float64))
        assert abs(np.linalg.norm(x) - 1) < 1e-5
        assert 1 - abs(x @ vt[3]) < (64 * np.finfo(np.float32).eps * s[0] / (s[2] - s[3])) ** 2 + 1e-6
    assert np.array_equal(np.abs(pynp.svd4_null(np.diag([3, 2, 2, 1]).astype(np.float32))), [0, 0, 0, 1])
    assert np.array_equal(np.abs(pynp.svd4_null(np.diag([3, 1, 2, 1]).astype(np.float32))), [0, 0, 0, 1])   # ties: the higher column


def test_every_reachable_verdict_occurs():
    seen = np.zeros(len(V), np.int64)
    for seed in (3, 4, 5):
        sc = sm.make_new_points_scene(n_nb=20, n=1000, seed=seed, zero_baseline_nb=5, no_shared_nb=7)
        seen += np.bincount(host(sc)[2].ravel(), minlength=len(V))
    # w == 0 needs an exactly singular pencil and dist == 0 a point on a camera centre, which the depth gates reject first; a
    # reprojection error in the neighbour above its gate while the line gate (same sigma, 3.84 < 5.991) passed did not occur either
    for name in ("none", "accepted", "parallax", "depth1", "depth2", "reproj1", "scale", "claimed"):
        assert seen[V[name]] > 0, name


def test_the_claim_rule():
    sc = sm.make_new_points_scene(n_nb=20, n=1000, seed=52)
    pts, b2, vd = host(sc)
    acc = vd == V["accepted"]
    assert (acc.sum(0) <= 1).all()                                   # one point per feature
    first = np.where(acc.any(0), acc.argmax(0), 99)
    nb = np.arange(20)[:, None]
    assert (vd[nb > first[None, :]] == V["claimed"]).all() and (b2[nb > first[None, :]] == -1).all()
    assert not (vd[nb <= first[None, :]] == V["claimed"]).any()
    rejected = (vd >= V["parallax"]) & (vd <= V["scale"])
    later = np.array([[(b2[b + 1:, i] >= 0).any() for i in range(1000)] for b in range(20)])
    assert (rejected & later).any()                                  # a feature rejected in one neighbour is tried again in a later one
    # the oracle with a rejected pair claiming its feature must differ here
    assert pynp.oracle(sc["cur"], sc["neighbours"], mutate=1)[0].tobytes() != pts.tobytes()


def test_two_features_may_share_one_idx2_and_the_order_is_the_references():
    sc = sm.make_new_points_scene(n_nb=10, n=800, seed=53)
    pts = host(sc)[0]
    key = pts["nb"].astype(np.int64) * 100000 + pts["idx2"]
    assert len(np.unique(key)) < len(key)                            # both points are reported
    order = pts["nb"].astype(np.int64) * 100000 + pts["idx1"]
    assert (np.diff(order) > 0).all()                                # neighbour ascending, idx1 ascending within one


def test_ties_replace_the_incumbent():
    for seed in range(54, 64):
        sc = sm.make_new_points_scene(n_nb=1, n=40, seed=seed, n_nodes=1, has_mp_frac=0.0, outlier_frac=0, octave_jump_frac=0, cross_frac=0,
                                      decoy_frac=0, twin_frac=0, tie_frac=0)
        c, v = sc["cur"], sc["neighbours"][0]
        b2 = host(sc)[1][0]
        hit = np.flatnonzero(b2 >= 0)
        if len(hit) == 0:
            continue
        i, j = int(hit[0]), int(b2[hit[0]])
        others = [k for k in range(40) if k != j][:2]
        lo, hi = min(others), max(others + [j])
        for k in others:                                             # two exact copies of the winner, before and after it
            for key in ("desc", "kp_xy", "octave"):
                v[key][k] = v[key][j]
        got = host(sc)[1][0][i]
        assert got == hi and got != lo                               # `>` keeps the last minimum; `>=` or first-wins would give lo
        same(host(sc), pynp.oracle(sc["cur"], sc["neighbours"]))
        return
    pytest.fail("no scene with a match")


def test_capacity_short_by_one_writes_nothing_but_the_count():
    sc = sm.make_new_points_scene(n_nb=6, n=500, seed=55)
    pts = host(sc)[0]
    with pytest.raises(api.CCMError, match="capacity %d below the %d points needed" % (len(pts) - 1, len(pts))) as e:
        host(sc, capacity=len(pts) - 1)
    assert e.value.needed == len(pts)
    assert host(sc, capacity=len(pts))[0].tobytes() == pts.tobytes()


def test_empty_inputs():
    sc = sm.make_new_points_scene(n_nb=3, n=200, seed=56)
    assert len(api.new_map_points(sc["cur"], [], host=True)) == 0
    full = sm.make_new_points_scene(n_nb=3, n=200, seed=56, all_have_mp=True)
    pts, b2, vd = host(full)
    assert len(pts) == 0 and (b2 == -1).all() and (vd == V["none"]).all()
    lone = sm.make_new_points_scene(n_nb=1, n=200, seed=57, no_shared_nb=0)
    assert len(host(lone)[0]) == 0


def bad(sc, match):
    with pytest.raises(api.CCMError, match=match):
        host(sc)


def test_validation_messages_name_the_neighbour():
    def fresh():
        sc = sm.make_new_points_scene(n_nb=3, n=120, seed=58)
        for v in [sc["cur"]] + sc["neighbours"]:
            for k in ("octave", "Tcw", "Ow", "node"):
                v[k] = v[k].copy()
        return sc
    sc = fresh(); sc["neighbours"][1]["octave"][7] = 8
    bad(sc, "neighbour 1: octave of feature 7 out of range")
    sc = fresh(); sc["cur"]["octave"][3] = -1
    bad(sc, "current keyframe: octave of feature 3 out of range")
    sc = fresh(); sc["neighbours"][2]["Tcw"][1, 3] = np.nan
    bad(sc, "neighbour 2: non-finite Tcw")
    sc = fresh(); sc["cur"]["Ow"][0] = np.inf
    bad(sc, "current keyframe: non-finite Ow")
    sc = fresh(); sc["neighbours"][0]["fv_feat"] = np.full(120, 120, np.uint32)
    bad(sc, "neighbour 0: bad FeatureVector: feature 120 out of range")
    sc = fresh(); sc["cur"]["fv_feat"] = np.zeros(120, np.uint32)
    bad(sc, "current keyframe: bad FeatureVector: feature 0 listed twice")
    sc = fresh(); sc["neighbours"][1]["fv_node_id"] = np.zeros(len(np.unique(sc["neighbours"][1]["node"])), np.uint32)
    bad(sc, "neighbour 1: bad FeatureVector: node ids are not ascending")
    keep = []
    c, nbs = api.new_points_structs(sc["cur"], fresh()["neighbours"], keep)
    n_out = api.C.c_int32()
    L = api.lib()
    assert L.ccm_new_map_points_host(None, nbs, 3, None, 0, api.C.byref(n_out), None, None) != 0
    assert L.ccm_new_map_points_host(api.C.byref(c), None, 3, None, 0, api.C.byref(n_out), None, None) != 0
    assert b"null neighbour array" in L.ccm_last_error()
    assert L.ccm_new_map_points_host(api.C.byref(c), nbs, -1, None, 0, api.C.byref(n_out), None, None) != 0
    assert b"negative size" in L.ccm_last_error()
    assert L.ccm_new_map_points_host(api.C.byref(c), nbs, 65536, None, 0, api.C.byref(n_out), None, None) != 0
    assert b"more than 65535 neighbours" in L.ccm_last_error()


def empty_nodes_scene():
    """the current keyframe's FeatureVector names its nodes but lists no feature under any of them"""
    sc = sm.make_new_points_scene(n_nb=2, n=100, seed=59)
    sc["cur"]["fv_node_ptr"] = np.zeros(len(np.unique(sc["cur"]["node"])) + 1, np.int32)
    sc["cur"]["fv_feat"] = np.zeros(0, np.uint32)
    return sc


def test_a_feature_vector_of_empty_nodes_gives_no_point():
    pts, b2, vd = host(empty_nodes_scene())
    assert len(pts) == 0 and (b2 == -1).all() and (vd == V["none"]).all()


# ---- hand-built pairs for the verdicts the generated scenes do not reach ----------------------------------------------------------
def single_pair_scene(kind):
    """One feature in the current keyframe and one in a single neighbour, cut from an accepted pair of a generated scene.  F12 is
    replaced by a matrix whose epipolar line is x = x2 whatever the current feature, and the epipole is moved far away, so the matcher
    pairs the two whatever is done to them next:
      reproj2    the current feature on the coarsest level, the neighbour's on the finest and moved 8 px: the error passes the
                 current keyframe's gate and fails the neighbour's
      dist_zero  the neighbour's camera centre Ow set to the bits of the triangulated point (Ow is an input of its own)"""
    sc = sm.make_new_points_scene(n_nb=1, n=60, seed=81, has_mp_frac=0.0, outlier_frac=0, octave_jump_frac=0, cross_frac=0, decoy_frac=0,
                                  twin_frac=0, tie_frac=0)
    pts = host(sc)[0]
    p = pts[len(pts) // 2]

    def cut(v, k):
        w = {key: (np.array(v[key][k:k + 1]) if key in ("desc", "has_mp", "kp_xy", "octave", "angle", "node") else v[key]) for key in VIEW_KEYS}
        w["node"] = np.zeros(1, np.int64); w["has_mp"] = np.zeros(1, np.uint8)
        return w
    c, v = cut(sc["cur"], p["idx1"]), cut(sc["neighbours"][0], p["idx2"])
    v["Ow"] = v["Ow"].copy()
    if kind == "reproj2":
        c["octave"][0] = 7; v["octave"][0] = 0
        v["kp_xy"][0, 1] += np.float32(8.0)
    elif kind == "dist_zero":
        v["Ow"][:] = p["x3D"]
    v["F12"] = np.array([[0, 0, 0], [0, 0, 0], [1, 0, -v["kp_xy"][0, 0]]], np.float32)
    v["ex"], v["ey"] = np.float32(1e6), np.float32(1e6)
    return dict(cur=c, neighbours=[v])


@pytest.mark.parametrize("kind", ["reproj2", "dist_zero"])
def test_hand_built_pairs_reach_the_remaining_verdicts(kind):
    sc = single_pair_scene(kind)
    got = host(sc)
    same(got, pynp.oracle(sc["cur"], sc["neighbours"]))
    assert got[1][0, 0] == 0 and got[2][0, 0] == V[kind] and len(got[0]) == 0
