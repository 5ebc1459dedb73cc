"""CPU suite: the Sim3 correction pass of a loop closure or a map merge (LoopFinder::CorrectLoop, cslam/src/LoopFinder.cpp:568-613;
MapMerger::MergeMaps, cslam/src/MapMerger.cpp:349-395) behind ccm_sim3_correction.

 * the pin: tests/golden/sim3_correction.npz, written by a witness (f64 scalar Sim3 operations in Eigen's order, cv2 for the f32 pose
   products and the normals) that its generator checks against the oracle; the oracle, the host entry point and the g++ build of
   sim3_correction_math.cuh all reproduce it bit for bit, NaN as NaN;
 * the three agree on seeded loop and merge scenes and on every edge-case knob;
 * the two order rules of the reference loop (the claim, the centres a normal reads) hold, and each deliberately wrong variant of the
   arithmetic (tests/host/sim3_correction_host.cpp -DMUT=n) is told apart;
 * the explicitly rounded Sim3 operations equal sim3_math.cuh's on the host;
 * refused input: the message names the entry, slot or point, and nothing is written.
The device kernels are tests/test_gpu_sim3_correction.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from ccm_slam_b200 import api, synth
from oracle import pysc

CCM_ERR_INVALID = -1
HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "host", "sim3_correction_host.cpp")
OUT = ("entry_Tcw", "entry_centre", "mp_entry", "mp_pos", "normal", "max_dist", "min_dist", "status")
EDGES = dict(K=24, P=700, window=6, null_frac=0.1, dup_frac=0.1, bad_mp_frac=0.05, tagged_frac=0.05, bad_kf_frac=0.3, all_bad_frac=0.08,
             off_ref_frac=0.3, no_ref_frac=0.03, empty_frac=0.15, null_entry_frac=0.15, unlisted_frac=0.05)
SCENES = {"loop": dict(kind="loop", seed=81, K=120, P=3000, n_loop=30, unlisted_frac=0.1), "merge": dict(kind="merge", seed=82, K=60, P=2500),
          "loop_edges": dict(kind="loop", seed=83, n_loop=9, **EDGES), "merge_edges": dict(kind="merge", seed=84, **EDGES),
          "merge_small": dict(kind="merge", p="small", seed=85), "loop_small": dict(kind="loop", p="small", seed=86, n_loop=12)}


def scene(kw):
    kw = dict(kw)
    p = kw.pop("p", None)
    return synth.make_sim3_correction(synth.make_config(p) if p else None, **kw)


def same(a, b):
    for k in OUT:
        assert np.array_equal(a[k], b[k], equal_nan=True), k


def _compile(tmp, mut):
    so = str(tmp / ("libsc_host_%d.so" % mut))
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-w", "-DMUT=%d" % mut,
                           "-o", so, SRC])
    return C.CDLL(so)


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    return _compile(tmp_path_factory.mktemp("sc"), 0)


def _fixture():
    z = np.load(os.path.join(HERE, "golden", "sim3_correction.npz"))
    n = len({k.split("_")[0] for k in z.files})
    for c in range(n):
        sc = {k: z["case%d_in_%s" % (c, k)] for k, _ in api.SIM3_CORRECTION_IN}
        yield sc, {k: z["case%d_%s" % (c, k)] for k in OUT}


def test_everything_reproduces_the_fixture(host):
    n = 0
    for sc, w in _fixture():
        same(pysc.oracle(sc), w)
        same(api.sim3_correction(sc, host=True), w)
        same(pysc.oracle(sc, fn=host.sc_host_correct), w)
        assert (w["mp_entry"] >= 0).sum() > 300
        n += 1
    assert n == 5


@pytest.mark.parametrize("name", list(SCENES))
def test_oracle_host_and_header_agree(host, name):
    sc = scene(SCENES[name])
    o = pysc.oracle(sc)
    same(api.sim3_correction(sc, host=True), o)
    same(pysc.oracle(sc, fn=host.sc_host_correct), o)
    assert (o["mp_entry"] >= 0).sum() > 100


def _first_lister(sc):
    """the claim rule restated on the flat arrays: the first entry in map order that lists a point not skipped"""
    first = np.full(len(sc["mp_skip"]), -1, np.int64)
    for e in range(len(sc["entry_kf"]) - 1, -1, -1):
        s = sc["slot_mp"][sc["slot_ptr"][e]:sc["slot_ptr"][e + 1]]
        s = s[s >= 0]
        first[s[sc["mp_skip"][s] == 0]] = e
    return first


@pytest.mark.parametrize("name", ["loop", "loop_edges", "merge_edges"])
def test_the_claim_and_the_knobs(name):
    sc = scene(SCENES[name])
    r = api.sim3_correction(sc, host=True)
    first = _first_lister(sc)
    assert np.array_equal(r["mp_entry"], first)
    moved = first >= 0
    assert (r["mp_pos"][~moved] == sc["mp_pos"][~moved]).all() and (r["status"][~moved] == 0).all()
    assert (r["mp_pos"][moved] != sc["mp_pos"][moved]).any(1).all()
    # points listed by several entries; some claimed by an entry that is not the lowest keyframe row among them
    E = len(sc["entry_kf"]); ptr = sc["slot_ptr"]
    ent = np.repeat(np.arange(E), np.diff(ptr)); mp = sc["slot_mp"]
    live = (mp >= 0) & (sc["mp_skip"][np.maximum(mp, 0)] == 0)
    low_row = np.full(len(first), np.iinfo(np.int32).max); np.minimum.at(low_row, mp[live], sc["entry_kf"][ent[live]])
    assert (moved & (sc["entry_kf"][np.maximum(first, 0)] != low_row)).sum() > 10
    # skipped points listed by an entry stay where they are
    listed = np.zeros(len(first), bool); listed[mp[mp >= 0]] = True
    assert (listed & (sc["mp_skip"] == 1)).sum() > 3
    if name == "merge_edges":
        assert (np.diff(ptr) == 0).any()                                    # an entry with no slots
        assert any((mp[ptr[e]:ptr[e + 1]] == -1).all() and ptr[e + 1] > ptr[e] for e in range(E))   # an entry whose slots are all null
        assert np.isnan(r["normal"][moved]).any(1).sum() > 3                # every observer bad
        assert (moved & (r["status"] == 0)).sum() > 0                       # no reference keyframe: the members stay as they were


def test_the_centres_a_normal_reads():
    """observers and reference keyframes of moved points are entries before, on and after the claiming entry and keyframes outside
    the list; the normals equal ccm_normal_depth_host's over a table that mixes corrected and pre-loop centres by that rule"""
    sc = scene(SCENES["loop"])
    r = api.sim3_correction(sc, host=True)
    K = len(sc["kf_bad"]); E = len(sc["entry_kf"])
    kf_entry = np.full(K, -1); kf_entry[sc["entry_kf"]] = np.arange(E)
    seen = {"before": 0, "on": 0, "after": 0, "outside": 0}
    ptr = sc["obs_ptr"]
    for c in range(E):
        pts = np.flatnonzero(r["mp_entry"] == c)
        if not len(pts):
            continue
        table = sc["kf_centre"].copy()
        before = sc["entry_kf"][:c]
        table[before] = r["entry_centre"][:c]
        sub = dict(kf_centre=table, kf_bad=sc["kf_bad"], mp_pos=r["mp_pos"][pts], mp_ref=sc["mp_ref"][pts], mp_scale_ref=sc["mp_scale_ref"][pts],
                   mp_scale_last=sc["mp_scale_last"][pts])
        deg = ptr[pts + 1] - ptr[pts]
        sub["obs_ptr"] = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
        sub["obs_kf"] = np.concatenate([sc["obs_kf"][ptr[i]:ptr[i + 1]] for i in pts]).astype(np.int32)
        nd = api.normal_depth(sub, host=True)
        for k in ("normal", "max_dist", "min_dist", "status"):
            assert np.array_equal(nd[k], r[k][pts], equal_nan=True), (c, k)
        e = np.concatenate([kf_entry[sub["obs_kf"]], kf_entry[sub["mp_ref"][sub["mp_ref"] >= 0]]])
        seen["before"] += int(((e >= 0) & (e < c)).sum()); seen["on"] += int((e == c).sum())
        seen["after"] += int((e > c).sum()); seen["outside"] += int((e < 0).sum())
    assert min(seen.values()) > 20, seen


@pytest.mark.parametrize("mut", range(1, 9))
def test_each_wrong_variant_is_told_apart(tmp_path, mut):
    lib = _compile(tmp_path, mut)
    differs = 0
    for sc, w in _fixture():
        m = pysc.oracle(sc, fn=lib.sc_host_correct)
        differs += sum(not np.array_equal(m[k], w[k], equal_nan=True) for k in OUT)
    assert differs > 0


def test_rounded_ops_equal_sim3_math(host):
    rng = np.random.default_rng(3)
    n = 4000
    q = rng.normal(size=(n, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True)
    q *= 1 + rng.normal(0, 1e-8, (n, 1))                              # not quite unit, as Eigen's quaternion from an f32 matrix
    S = np.concatenate([q, rng.normal(0, 5, (n, 3)), rng.uniform(0.3, 3, (n, 1))], 1)
    x = rng.normal(0, 20, (n, 3))
    out = np.zeros((n, 4, 8)); R = np.zeros((n, 2, 9))
    host.sc_host_ops(n, S.ctypes.data_as(C.c_void_p), x.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p), R.ctypes.data_as(C.c_void_p))
    assert np.array_equal(out[:, 0], out[:, 1]) and np.array_equal(out[:, 2, :3], out[:, 3, :3]) and np.array_equal(R[:, 0], R[:, 1])
    assert not np.array_equal(out[:, 0], np.zeros((n, 8)))


def _refused(sc, msg):
    for host in (True, False):                                             # validation runs before the device is looked for
        out = api.sim3_correction_out(len(sc["entry_kf"]), len(sc["mp_skip"]))
        for v in out.values():
            v.fill(7)
        with pytest.raises(api.CCMError) as ei:
            api.sim3_correction(sc, host=host, out=out)
        assert ei.value.code == CCM_ERR_INVALID
        assert msg in str(ei.value), str(ei.value)
        for v in out.values():
            assert (v == 7).all()


def test_refused_input_names_the_culprit_and_writes_nothing():
    base = scene(SCENES["loop_edges"])
    sc = dict(base); sc["entry_kf"] = base["entry_kf"].copy(); sc["entry_kf"][2] = 99
    _refused(sc, "entry 2: keyframe row 99 out of range")
    sc = dict(base); sc["entry_kf"] = base["entry_kf"].copy(); sc["entry_kf"][3] = sc["entry_kf"][1]
    _refused(sc, "entry 3: keyframe row %d is already entry 1" % base["entry_kf"][1])
    sc = dict(base); sc["slot_mp"] = base["slot_mp"].copy()
    e = int(np.flatnonzero(np.diff(base["slot_ptr"]) > 2)[0]); sc["slot_mp"][base["slot_ptr"][e] + 2] = len(base["mp_skip"])
    _refused(sc, "entry %d, slot 2: point row %d out of range" % (e, len(base["mp_skip"])))
    sc = dict(base); sc["obs_kf"] = base["obs_kf"].copy(); sc["obs_kf"][-1] = -3
    _refused(sc, "point %d: observer row -3 out of range" % (len(base["mp_skip"]) - 1))
    sc = dict(base); sc["mp_ref"] = base["mp_ref"].copy(); sc["mp_ref"][5] = 1000
    _refused(sc, "point 5: reference row 1000 out of range")


def test_null_arrays_are_refused():
    sc = scene(SCENES["merge_edges"])
    out = api.sim3_correction_out(len(sc["entry_kf"]), len(sc["mp_skip"]))
    argv, _keep = api.sim3_correction_args(sc, out)
    for i, what in ((1, "null keyframe array"), (5, "null entry array"), (8, "null slot_mp"), (11, "null point array"), (13, "null obs_kf"),
                    (20, "null point array")):
        a = list(argv); a[i] = None
        for fn in (api.lib().ccm_sim3_correction_host, api.lib().ccm_sim3_correction):
            assert fn(*a) == CCM_ERR_INVALID
            assert what in api.lib().ccm_last_error().decode()


def test_empty_inputs():
    sc = scene(dict(kind="merge", seed=87, K=6, P=50))
    e = dict(sc); e["entry_kf"] = sc["entry_kf"][:0]; e["entry_Siw_new"] = sc["entry_Siw_new"][:0]; e["entry_Siw_old"] = sc["entry_Siw_old"][:0]
    e["slot_ptr"] = np.zeros(1, np.int64); e["slot_mp"] = np.zeros(0, np.int32)
    r = api.sim3_correction(e, host=True)
    same(r, pysc.oracle(e))
    assert (r["mp_entry"] == -1).all() and np.array_equal(r["mp_pos"], sc["mp_pos"])
