"""shim/KeyFrameCulling_shim.cpp (LocalMapping::KeyFrameCullingV3 over one ccm_keyframe_culling call) against a literal restatement of
the member and of the SetBadFlag / EraseObservation paths it reaches (oracle/ref_keyframe_culling_wrap.cpp), member for member on
stand-in objects: every keyframe's mbBad, mbToBeErased and mvpMapPoints, every point's mbBad, nObs, mpRefKF and observations,
mCulledKfs and mspKFsCheckedForCulling, on scenes with cascades.  The device entry point is answered by the host entry point here;
tests/test_gpu_keyframe_culling.py runs the same over the real library."""
import numpy as np
import pytest

from ccm_slam_b200 import synth
from oracle import pykc

KEYS = ("kf_bad", "to_be_erased", "slots", "mp_bad", "nobs", "ref", "obs_ptr", "obs", "culled", "checked")
SCENES = {"server20": dict(n_c=20, slots=600, seed=21), "server60": dict(n_c=60, slots=300, seed=22, n_redundant=5),
          "edges": dict(n_c=10, slots=200, seed=23, obs=(3, 8), bad_kf_frac=0.2, no_ref_frac=0.05, dup_frac=0.05, null_frac=0.1,
                        n_redundant=4),
          "cascades_only": dict(n_c=0, seed=24)}


def run_both(sc, gpu=False, **kw):
    out, stats = [], None
    for mode in (0, 1):
        s = pykc.StandIn(sc, gpu=gpu, **kw)
        before = s.stats()
        s.run(mode)
        out.append(s.members())
        if mode == 1:
            stats = s.stats() - before
        s.close()
    return out[0], out[1], stats


def same_members(a, b):
    for k in KEYS:
        assert a[k].tobytes() == b[k].tobytes(), k


def compare(name, gpu=False):
    sc = synth.make_keyframe_culling_scene(**SCENES[name])
    ref, shim, stats = run_both(sc, gpu=gpu)
    same_members(ref, shim)
    assert stats[0] == 1 and stats[1] > 0                         # one library call; candidates counted again after a cull
    assert ref["culled"][0] >= 3                                  # mCulledKfs, culls without effect included
    assert (ref["to_be_erased"] == 1).any()                       # a redundant candidate with mbNotErase
    assert ref["mp_bad"].sum() > sc["mp_bad"].sum()               # culls turned points bad
    return ref


@pytest.mark.parametrize("name", list(SCENES))
def test_shim_equals_restatement(name):
    compare(name)


def test_pick_rules_are_kept():
    sc = synth.make_keyframe_culling_scene(n_c=5, slots=100, seed=25)
    q, r = int(sc["query"]), int(sc["recent"][0])
    for picks, checked, runs in (([-1], (), False), ([r, r], (), False), ([r, q], (), True), ([q], (q,), False), ([r, -1], (), False)):
        ref, shim, stats = run_both(sc, picks=picks, checked=checked)
        same_members(ref, shim)
        assert stats[0] == int(runs)
        assert (ref["culled"][0] > 0) == runs
        assert ref["checked"][q] == int(runs or q in checked)
