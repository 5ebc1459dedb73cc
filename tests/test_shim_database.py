"""shim/Database_shim.cpp (cslam::KeyFrameDatabase over ccm_kfdb_*, compiled against the reference's own cslam/Database.h) side by
side with the reference's own Database.cpp, on the same stand-in KeyFrame / Map / Frame records and every scene of tests/kfdb_scenes.py:
the returned vector<kfptr> is identical, and the marker members of the scored candidates are the reference's, bit for bit.

CPU: oracle/_ref/libkfdb_shim.so, the device entry points doubled by oracle/ccm_kfdb_double.cpp.
GPU: oracle/_ref/libkfdb_shim_gpu.so over the real library."""
import numpy as np
import pytest

from oracle import pykfdb
from tests.kfdb_scenes import SCORINGS, all_scenes, replay_checker

SCENES = all_scenes()
_MARK = {"loop": (0, 0, 0), "mm": (1, 0, 0), "reloc": (2, 1, 1)}   # (query-id marker, count, score) index per kind


def _side_by_side(shim_cls, name, scoring, check_vectors=True):
    if not pykfdb.Reference.available() or not shim_cls.available():
        pytest.skip("oracle/_ref/libkfdb_ref.so / the shim library are not built (need the reference tree and the product at build time)")
    scene = SCENES[name]
    runs = zip(replay_checker(scene, scoring, pykfdb.Oracle), replay_checker(scene, scoring, pykfdb.Reference),
               replay_checker(scene, scoring, shim_cls))
    n_queries = 0
    for (op, r0, o), (_, r1, ref), (_, r2, shim) in runs:
        if r1 is None:
            continue
        n_queries += 1
        if check_vectors:
            assert r2.tolist() == r1.tolist(), (name, scoring, op)
        qi, ci, si = _MARK[op[0]]
        for u in o.last_scored()["uid"].tolist():
            m1, m2 = ref.markers(u), shim.markers(u)
            assert m2[0][qi] == m1[0][qi] and m2[1][ci] == m1[1][ci], (name, op, u)
            if check_vectors:
                assert m2[2][si:si + 1].view(np.uint32)[0] == m1[2][si:si + 1].view(np.uint32)[0], (name, op, u)
    assert n_queries > 0


@pytest.mark.parametrize("scoring", SCORINGS)
@pytest.mark.parametrize("name", sorted(SCENES))
def test_shim_equals_the_reference_database(name, scoring):
    _side_by_side(pykfdb.Shim, name, scoring)


@pytest.mark.gpu
@pytest.mark.parametrize("scoring", SCORINGS)
def test_shim_over_the_device_equals_the_reference_database(scoring):
    from ccm_slam_b200 import api
    api.init(0)
    for name in sorted(SCENES):
        _side_by_side(pykfdb.ShimGPU, name, scoring, check_vectors=scoring != 3)   # KL: the device log (DESIGN.md §5)
