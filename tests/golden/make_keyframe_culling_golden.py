"""Generates tests/golden/keyframe_culling.npz: LocalMapping::KeyFrameCullingV3 (cslam/src/Mapping.cpp:771-863) evaluated by a witness
written here, on the map scenes of synth.make_keyframe_culling_scene.  The witness walks the member literally over mutable Python state:
per keyframe its bad flag and its mvpMapPoints list, per point its bad flag, nObs, mpRefKF and an ordered dict of observations; it
restates KeyFrame::SetBadFlag (KeyFrame.cpp:936-990, the server's mbNotErase branch), MapPoint::EraseObservation (MapPoint.cpp:442-509)
and MapPoint::SetBadFlag (which nulls the point in every observer's slots) and calls them the moment a verdict is reached.

The f64 / f32 case is found by search: the first (threshold, nMPs, nRedundant) in a fixed order for which `nRed > thres * nMPs` in
f64 and the same expression in f32 disagree (none exists for 0.98 below 5000 points).  Before it writes, every case is checked against
the oracle (oracle/keyframe_culling_oracle.cpp); the generator refuses to write on any difference.  Inputs and outputs are both
stored, so the fixture does not depend on the generator's random streams.  Run from the repo root:
    python tests/golden/make_keyframe_culling_golden.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
from ccm_slam_b200 import api, synth  # noqa: E402

INPUTS = [k for k, _ in api.KEYFRAME_CULLING_IN] + ["th_obs", "red_thres"]
OUTPUTS = ("cull", "n_mps", "n_red")
CASES = [dict(n_c=20, slots=1000, seed=11),
         dict(n_c=40, slots=500, seed=12, n_redundant=4),
         dict(n_c=8, slots=300, seed=13, obs=(3, 8), bad_kf_frac=0.2, no_ref_frac=0.05, dup_frac=0.05, null_frac=0.1, n_redundant=3),
         "split"]


def find_split():
    """(threshold, nMPs, nRedundant) where the f64 and the f32 readings of the member's comparison disagree"""
    for thres in (0.98, 0.95, 0.9, 0.8, 0.75, 0.7, 0.6, 0.5):
        t32 = np.float32(thres)
        for n in range(1, 2001):
            for k in range(max(0, int(thres * n) - 1), min(n, int(thres * n) + 1) + 1):
                if (k > thres * n) != bool(np.float32(k) > t32 * np.float32(n)):
                    return thres, n, k
    raise SystemExit("no f64 / f32 split found")


def witness(sc):
    K = len(sc["kf_bad"])
    sptr, smp, soct = sc["kf_slot_ptr"], sc["kf_slot_mp"], sc["kf_slot_octave"]
    kf_bad = [bool(b) for b in sc["kf_bad"]]
    slots = [[int(p) for p in smp[sptr[k]:sptr[k + 1]]] for k in range(K)]
    octave = lambda k, i: int(soct[sptr[k] + i])  # noqa: E731
    mp_bad = [bool(b) for b in sc["mp_bad"]]
    nobs = [int(n) for n in sc["mp_nobs"]]
    ref = [int(r) for r in sc["mp_ref"]]
    obs = [{int(sc["obs_kf"][j]): int(sc["obs_idx"][j]) for j in range(sc["obs_ptr"][p], sc["obs_ptr"][p + 1])} for p in range(len(nobs))]
    th, thres = int(sc["th_obs"]), float(sc["red_thres"])

    def mp_set_bad(p):                       # MapPoint::SetBadFlag
        if mp_bad[p]:
            return
        mp_bad[p] = True
        o, obs[p] = obs[p], {}
        for k, idx in o.items():
            slots[k][idx] = -1                # pKF->EraseMapPointMatch(idx)

    def erase_observation(p, k):             # MapPoint::EraseObservation(pKF, false, true), server
        bad = False
        if k in obs[p]:
            nobs[p] -= 1
            del obs[p][k]
            if ref[p] == k:
                ref[p] = -1
                if nobs[p] > 0:
                    for kk in obs[p]:
                        if not kf_bad[kk]:
                            ref[p] = kk
                            break
            if nobs[p] <= 2:
                bad = True
        if bad:
            mp_set_bad(p)
        if ref[p] < 0 and not mp_bad[p]:
            mp_set_bad(p)

    def kf_set_bad(k, not_erase):            # KeyFrame::SetBadFlag, server; mId.first 0 never reaches it
        if kf_bad[k] or not_erase:
            return
        for i in range(len(slots[k])):
            if slots[k][i] >= 0:
                erase_observation(slots[k][i], k)
        kf_bad[k] = True

    out = dict(cull=[], n_mps=[], n_red=[])
    recent = set(int(r) for r in sc["recent"])
    for pKF in (int(k) for k in sc["covis"]):
        if sc["kf_id"][pKF] in (0, 1) or pKF in recent:
            continue
        vp = list(slots[pKF])
        n_red = n_mps = 0
        for i, p in enumerate(vp):
            if p < 0 or mp_bad[p]:
                continue
            n_mps += 1
            if nobs[p] > th:
                level = octave(pKF, i)
                n = 0
                for k, idx in list(obs[p].items()):
                    if kf_bad[k] or k == pKF:
                        continue
                    if octave(k, idx) <= level + 1:
                        n += 1
                        if n >= th:
                            break
                if n >= th:
                    n_red += 1
        cull = n_red > thres * n_mps
        out["cull"].append(cull); out["n_mps"].append(n_mps); out["n_red"].append(n_red)
        if cull:
            kf_set_bad(pKF, bool(sc["kf_not_erase"][pKF]))
    return dict(cull=np.asarray(out["cull"], np.uint8), n_mps=np.asarray(out["n_mps"], np.int32), n_red=np.asarray(out["n_red"], np.int32))


def scene(kw):
    if kw == "split":
        thres, n, k = find_split()
        return synth.make_keyframe_culling_scene(n_c=0, seed=14, split=(n, k), edges=False, red_thres=thres)
    return synth.make_keyframe_culling_scene(**kw)


def main():
    from oracle import pykc
    z = {}
    for c, kw in enumerate(CASES):
        sc = scene(kw)
        w = witness(sc)
        o = pykc.oracle(sc)
        for k in OUTPUTS:
            if not np.array_equal(w[k], o[k]):
                raise SystemExit("case %d: witness and oracle differ in %s; not writing" % (c, k))
        for k in INPUTS:
            z["case%d_in_%s" % (c, k)] = np.asarray(sc[k])
        for k in OUTPUTS:
            z["case%d_%s" % (c, k)] = w[k]
        print("case %d: %d candidates, %d slots, %d culls, threshold %r" % (c, len(sc["cand_kf"]), sc["slot_ptr"][-1], w["cull"].sum(),
                                                                          sc["red_thres"]))
    np.savez_compressed(os.path.join(HERE, "keyframe_culling.npz"), **z)


if __name__ == "__main__":
    main()
