"""GPU suite: the per-thread staging of the batched entry points (Staging, ccm_slam_b200/csrc/common.cuh).  Blocks grown by a large
call and reused by smaller and larger ones, two threads calling at once, and a change of device give the bytes a fresh thread, the
host entry point and the CPU Hamming distances give."""
import threading

import numpy as np
import pytest

from ccm_slam_b200 import api, synth
from ccm_slam_b200 import synth_match as sm

pytestmark = pytest.mark.gpu

SIM3_OUT = ("entry_Tcw", "entry_centre", "mp_entry", "mp_pos", "normal", "max_dist", "min_dist", "status")


@pytest.fixture(scope="module", autouse=True)
def device():
    if api.device_count() == 0:
        pytest.skip("no CUDA device")
    api.init(0)


POPCOUNT = np.unpackbits(np.arange(256, dtype=np.uint8)[:, None], axis=1).sum(1).astype(np.uint16)


def hamming_cpu(A, B):
    return np.concatenate([POPCOUNT[A[i:i + 64, None, :] ^ B[None, :, :]].sum(2, dtype=np.uint16) for i in range(0, len(A), 64)])


def descriptors(n, seed):
    return np.random.default_rng(seed).integers(0, 256, (n, 32), dtype=np.uint8)


# each call returns its result arrays; host=True runs the host entry point (the CPU distances for hamming)
def run_sim3(sc, host=False):
    r = api.sim3_correction(sc, host=host)
    return [r[k] for k in SIM3_OUT]


def run_new_points(sc, host=False):
    return list(api.new_map_points(sc["cur"], sc["neighbours"], want_debug=True, host=host))


def run_fuse(sc, host=False):
    return list(api.fuse_neighbours(sc, host=host)[:2])


def run_search_and_fuse(sc, host=False):
    return [api.search_and_fuse(sc, host=host)[0]]


def run_hamming(sc, host=False):
    A, B = sc
    return [hamming_cpu(A, B) if host else api.hamming_matrix(A, B)]


RUN = dict(sim3=run_sim3, new_points=run_new_points, fuse=run_fuse, search_and_fuse=run_search_and_fuse, hamming=run_hamming)


# a large call, a small one, then one larger than the first
SIZES = (dict(K=200, P=20000, loop=30, nb=12, n_np=1000, nf=10, n_fu=1000, kf=12, n_sf=800, n_pts=4000, nA=1500, nB=1200),
         dict(K=12, P=300, loop=4, nb=2, n_np=300, nf=1, n_fu=200, kf=2, n_sf=200, n_pts=100, nA=40, nB=30),
         dict(K=300, P=40000, loop=60, nb=20, n_np=1500, nf=20, n_fu=1000, kf=31, n_sf=1000, n_pts=8000, nA=2000, nB=1800))


def scenes(z, seed):
    """one scene per staged entry point at sizes z"""
    return dict(sim3=synth.make_sim3_correction(kind="merge", seed=seed, K=z["K"], P=z["P"], n_loop=z["loop"]),
                new_points=sm.make_new_points_scene(n_nb=z["nb"], n=z["n_np"], seed=seed),
                fuse=sm.make_fuse_scene(n_first=z["nf"], n_second=z["nf"] // 4, n=z["n_fu"], seed=seed),
                search_and_fuse=sm.make_search_and_fuse_scene("loop", n_kf=z["kf"], n=z["n_sf"], n_loop=z["n_pts"], seed=seed),
                hamming=(descriptors(z["nA"], seed), descriptors(z["nB"], seed + 1)))


@pytest.fixture(scope="module")
def growth():
    return [scenes(z, seed=40 + i) for i, z in enumerate(SIZES)]


def on_fresh_thread(fn, *args):
    out = {}

    def body():
        try:
            out["r"] = fn(*args)
        except BaseException as e:   # re-raised on the calling thread
            out["e"] = e

    t = threading.Thread(target=body)
    t.start()
    t.join()
    if "e" in out:
        raise out["e"]
    return out["r"]


def interleaved(scs):
    """every entry point on each scene set in turn, on the calling thread, as bytes"""
    return [{name: as_bytes(RUN[name](sc[name])) for name in RUN} for sc in scs]


def as_bytes(arrays):
    return [a.tobytes() for a in arrays]


def equals_host(got, sc, name):
    """the host entry point's values; a NaN may carry another payload there (test_gpu_sim3_correction compares the same way)"""
    want = RUN[name](sc, host=True)
    return all(np.array_equal(np.frombuffer(g, w.dtype).reshape(w.shape), w, equal_nan=w.dtype.kind == "f")
               for g, w in zip(got, want)) and len(got) == len(want)


def test_growth_and_reuse_on_one_thread(growth):
    got = on_fresh_thread(interleaved, growth)
    for sc, res in zip(growth, got):
        for name in RUN:
            assert res[name] == as_bytes(on_fresh_thread(RUN[name], sc[name])), name
            assert equals_host(res[name], sc[name], name), name


def test_two_threads_at_once(growth):
    sets = [[growth[0], growth[1], growth[2]], [growth[2], growth[0], growth[1]]]
    serial = [interleaved(s) for s in sets]
    got = [None, None]
    errors = []
    barrier = threading.Barrier(2)

    def body(i):
        try:
            barrier.wait()
            got[i] = [interleaved(sets[i]) for _ in range(3)]
        except BaseException as e:
            errors.append(e)

    threads = [threading.Thread(target=body, args=(i,)) for i in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    if errors:
        raise errors[0]
    for i in range(2):
        for rep in got[i]:
            assert rep == serial[i]


def test_device_switch():
    if api.device_count() < 2:
        pytest.skip("needs two CUDA devices")
    A, B = descriptors(700, 1), descriptors(500, 2)
    sc = synth.make_sim3_correction(kind="loop", seed=5, K=60, P=3000)
    try:
        assert equals_host(as_bytes(run_hamming((A, B))), (A, B), "hamming")
        api.init(1)
        assert equals_host(as_bytes(run_hamming((A, B))), (A, B), "hamming")
        api.init(0)
        assert equals_host(as_bytes(run_sim3(sc)), sc, "sim3")
        api.init(1)
        assert equals_host(as_bytes(run_sim3(sc)), sc, "sim3")
    finally:
        api.init(0)
