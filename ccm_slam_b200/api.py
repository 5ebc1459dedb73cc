"""ctypes binding of libccm_b200.so — the thin Python face of the C ABI in include/ccm_b200.h.

This is host-side plumbing for tests and bench.py; the product is the shared library.  There is no CPU fallback:
if the library is missing, or no CUDA device is present, the calls raise.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libccm_b200.so")
TRACE_COLS = 8
_lib = None


class CCMError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"libccm_b200 error {code}: {msg}")
        self.code = code


class BAProblemC(C.Structure):
    _fields_ = [("K", C.c_int32), ("P", C.c_int32), ("E", C.c_int32),
                ("poses", C.c_void_p), ("intr", C.c_void_p), ("fixed", C.c_void_p), ("points", C.c_void_p),
                ("obs_kf", C.c_void_p), ("obs_mp", C.c_void_p), ("obs_uv", C.c_void_p), ("obs_w", C.c_void_p),
                ("edge_flags", C.c_void_p)]


class BAOptionsC(C.Structure):
    _fields_ = [("iterations", C.c_int32), ("robust", C.c_int32), ("huber_delta", C.c_double),
                ("lambda_init", C.c_double), ("max_trials", C.c_int32), ("pcg_max_iter", C.c_int32),
                ("pcg_tol", C.c_double), ("stop", C.c_void_p)]


class BAResultC(C.Structure):
    _fields_ = [("poses", C.c_void_p), ("points", C.c_void_p), ("chi2", C.c_void_p), ("depth_pos", C.c_void_p),
                ("trace", C.c_void_p), ("trace_cap", C.c_int32), ("trace_len", C.c_int32),
                ("iters_done", C.c_int32), ("trials_total", C.c_int32), ("pcg_iters_total", C.c_int32),
                ("pcg_not_converged", C.c_int32),
                ("chi2_initial", C.c_double), ("chi2_final", C.c_double), ("lambda_final", C.c_double),
                ("t_setup_ms", C.c_double), ("t_optimize_ms", C.c_double), ("t_download_ms", C.c_double),
                ("t_optimize_event_ms", C.c_double)]


class BAInfoC(C.Structure):
    _fields_ = [("K", C.c_int32), ("K_free", C.c_int32), ("P_local", C.c_int32), ("E_local", C.c_int32),
                ("rank", C.c_int32), ("nranks", C.c_int32), ("s_blocks_upper", C.c_int64),
                ("s_blocks_full", C.c_int64), ("schur_products", C.c_int64), ("device_bytes", C.c_int64)]


class PGOProblemC(C.Structure):
    _fields_ = [("K", C.c_int32), ("E", C.c_int32), ("sim3", C.c_void_p), ("fixed", C.c_void_p),
                ("edge_i", C.c_void_p), ("edge_j", C.c_void_p), ("meas", C.c_void_p), ("fix_scale", C.c_int32)]


class PGOOptionsC(C.Structure):
    _fields_ = [("iterations", C.c_int32), ("lambda_init", C.c_double), ("pcg_max_iter", C.c_int32),
                ("pcg_tol", C.c_double), ("stop", C.c_void_p)]


class PGOResultC(C.Structure):
    _fields_ = [("sim3", C.c_void_p), ("trace", C.c_void_p), ("trace_cap", C.c_int32), ("trace_len", C.c_int32),
                ("iters_done", C.c_int32), ("chi2_initial", C.c_double), ("chi2_final", C.c_double),
                ("lambda_final", C.c_double), ("t_total_ms", C.c_double)]


class ORBConfigC(C.Structure):
    _fields_ = [("nfeatures", C.c_int32), ("scale_factor", C.c_float), ("nlevels", C.c_int32),
                ("ini_th_fast", C.c_int32), ("min_th_fast", C.c_int32), ("blur_2413", C.c_int32)]


class KeyPointC(C.Structure):
    _fields_ = [("x", C.c_float), ("y", C.c_float), ("size", C.c_float), ("angle", C.c_float),
                ("response", C.c_float), ("octave", C.c_int32)]


class FeatureVectorC(C.Structure):
    _fields_ = [("n_nodes", C.c_int32), ("node_id", C.c_void_p), ("node_ptr", C.c_void_p), ("feat", C.c_void_p)]


class TriViewC(C.Structure):
    _fields_ = [("desc", C.c_void_p), ("n", C.c_int32), ("has_mp", C.c_void_p), ("kp_xy", C.c_void_p),
                ("octave", C.c_void_p), ("angle", C.c_void_p), ("fv", C.POINTER(FeatureVectorC)),
                ("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float), ("cy", C.c_float)]


def lib():
    """Loads the shared library; fails loudly when it has not been built (python ccm_slam_b200/build.py)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise CCMError(-100, f"{LIB_PATH} is missing: run `python ccm_slam_b200/build.py` (no CPU fallback exists)")
        _lib = C.CDLL(LIB_PATH)
        _lib.ccm_last_error.restype = C.c_char_p
        _lib.ccm_kernel_launches.restype = C.c_uint64
    return _lib


def _chk(rc):
    if rc != 0:
        raise CCMError(rc, lib().ccm_last_error().decode())


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def device_count() -> int:
    return lib().ccm_device_count()


def init(device: int = 0):
    _chk(lib().ccm_init(device))


def l2_flush():
    _chk(lib().ccm_l2_flush())


def host_register(arr: np.ndarray):
    _chk(lib().ccm_host_register(_p(arr), C.c_uint64(arr.nbytes)))


def host_unregister(arr: np.ndarray):
    _chk(lib().ccm_host_unregister(_p(arr)))


def kernel_launches() -> int:
    return int(lib().ccm_kernel_launches())


def comm_unique_id() -> np.ndarray:
    buf = np.zeros(128, np.uint8)
    _chk(lib().ccm_comm_unique_id(_p(buf)))
    return buf


def comm_init(rank: int, nranks: int, uid: np.ndarray):
    uid = np.ascontiguousarray(uid, np.uint8)
    _chk(lib().ccm_comm_init(rank, nranks, _p(uid)))


def comm_destroy():
    _chk(lib().ccm_comm_destroy())


def _ba_arrays(p):
    return dict(poses=np.ascontiguousarray(p.poses, np.float64), intr=np.ascontiguousarray(p.intr, np.float64),
                fixed=np.ascontiguousarray(p.fixed, np.uint8), points=np.ascontiguousarray(p.points, np.float64),
                obs_kf=np.ascontiguousarray(p.obs_kf, np.int32), obs_mp=np.ascontiguousarray(p.obs_mp, np.int32),
                obs_uv=np.ascontiguousarray(p.obs_uv, np.float32), obs_w=np.ascontiguousarray(p.obs_w, np.float32),
                edge_flags=None if p.edge_flags is None else np.ascontiguousarray(p.edge_flags, np.uint8))


def _ba_struct(arrs):
    return BAProblemC(arrs["poses"].shape[0], arrs["points"].shape[0], arrs["obs_kf"].shape[0],
                      *[_p(arrs[k]) for k in ("poses", "intr", "fixed", "points", "obs_kf", "obs_mp", "obs_uv", "obs_w", "edge_flags")])


def _ba_options(iterations, robust, huber_delta, lambda_init, max_trials, pcg_max_iter, pcg_tol, stop):
    return BAOptionsC(iterations, int(robust), float(huber_delta), float(lambda_init), max_trials, pcg_max_iter,
                      float(pcg_tol), _p(stop))


def _result_dict(res, poses, points, chi2, depth, trace):
    return dict(poses=poses, points=points, chi2=chi2, depth_pos=depth, trace=trace[:res.trace_len],
                iters_done=res.iters_done, trials_total=res.trials_total, pcg_iters_total=res.pcg_iters_total,
                pcg_not_converged=res.pcg_not_converged, chi2_initial=res.chi2_initial, chi2_final=res.chi2_final,
                lambda_final=res.lambda_final, t_setup_ms=res.t_setup_ms, t_optimize_ms=res.t_optimize_ms,
                t_download_ms=res.t_download_ms, t_optimize_event_ms=res.t_optimize_event_ms)


HUBER_GBA = float(np.float32(np.sqrt(5.99)))     # `const float thHuber2D = sqrt(5.99)`   S/Optimizer.cpp:712
HUBER_LOCAL = float(np.float32(np.sqrt(5.991)))  # `const float thHuberMono = sqrt(5.991)` S/Optimizer.cpp:468


def ba_solve(p, iterations=20, robust=True, huber_delta=HUBER_GBA, lambda_init=-1.0, max_trials=10,
             pcg_max_iter=0, pcg_tol=0.0, stop=None, chi2_in=None, want_edges=True):
    """One-shot ccm_ba_solve: host buffers in, host buffers out (upload + structure + LM + download)."""
    arrs = _ba_arrays(p)
    prob = _ba_struct(arrs)
    K, P, E = prob.K, prob.P, prob.E
    poses = np.empty((K, 7)); points = np.empty((P, 3))
    chi2 = (np.zeros(E) if chi2_in is None else np.array(chi2_in, np.float64)) if want_edges else None
    depth = np.zeros(E, np.uint8) if want_edges else None
    trace = np.zeros((max(iterations, 1), TRACE_COLS))
    opt = _ba_options(iterations, robust, huber_delta, lambda_init, max_trials, pcg_max_iter, pcg_tol, stop)
    res = BAResultC(_p(poses), _p(points), _p(chi2), _p(depth), _p(trace), trace.shape[0])
    _chk(lib().ccm_ba_solve(C.byref(prob), C.byref(opt), C.byref(res)))
    return _result_dict(res, poses, points, chi2, depth, trace)


class BAHandle:
    """ccm_ba_create / optimize / reset / destroy: the device-resident form used by LocalBA's two rounds and bench.py."""

    def __init__(self, p):
        self._arrs = _ba_arrays(p)
        prob = _ba_struct(self._arrs)
        self.K, self.P, self.E = prob.K, prob.P, prob.E
        self._h = C.c_void_p()
        _chk(lib().ccm_ba_create(C.byref(prob), C.byref(self._h)))

    def close(self):
        if self._h:
            lib().ccm_ba_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def reset(self):
        _chk(lib().ccm_ba_reset(self._h))

    def set_edge_flags(self, flags):
        f = None if flags is None else np.ascontiguousarray(flags, np.uint8)
        _chk(lib().ccm_ba_set_edge_flags(self._h, _p(f)))

    def info(self):
        i = BAInfoC()
        _chk(lib().ccm_ba_get_info(self._h, C.byref(i)))
        return {k: getattr(i, k) for k, _ in BAInfoC._fields_}

    def optimize(self, iterations=20, robust=True, huber_delta=HUBER_GBA, lambda_init=-1.0, max_trials=10,
                 pcg_max_iter=0, pcg_tol=0.0, stop=None, chi2_in=None, want_state=True, want_edges=False):
        poses = np.empty((self.K, 7)) if want_state else None
        points = np.empty((self.P, 3)) if want_state else None
        chi2 = (np.zeros(self.E) if chi2_in is None else np.array(chi2_in, np.float64)) if want_edges else None
        depth = np.zeros(self.E, np.uint8) if want_edges else None
        trace = np.zeros((max(iterations, 1), TRACE_COLS))
        opt = _ba_options(iterations, robust, huber_delta, lambda_init, max_trials, pcg_max_iter, pcg_tol, stop)
        res = BAResultC(_p(poses), _p(points), _p(chi2), _p(depth), _p(trace), trace.shape[0])
        _chk(lib().ccm_ba_optimize(self._h, C.byref(opt), C.byref(res)))
        return _result_dict(res, poses, points, chi2, depth, trace)

    KERNEL_NAMES = ["linearize", "pose_pass", "scale", "schur", "allreduce", "finalize", "pcg", "backsub", "residual"]

    def set_profile(self, on=True):
        _chk(lib().ccm_ba_set_profile(self._h, int(on)))

    def kernel_stats(self):
        ms = np.zeros(len(self.KERNEL_NAMES)); cnt = np.zeros(len(self.KERNEL_NAMES), np.int64)
        _chk(lib().ccm_ba_get_kernel_stats(self._h, _p(ms), _p(cnt)))
        return {n: dict(total_ms=float(ms[i]), launches=int(cnt[i])) for i, n in enumerate(self.KERNEL_NAMES)}

    def debug_build(self, robust=True, huber_delta=HUBER_GBA):
        Hpp = np.empty((self.K, 6, 6)); bp = np.empty((self.K, 6)); Hll = np.empty((self.P, 3, 3)); bl = np.empty((self.P, 3))
        W = np.empty((self.E, 6, 3)); chi = C.c_double()
        _chk(lib().ccm_ba_debug_build(self._h, int(robust), C.c_double(huber_delta), _p(Hpp), _p(bp), _p(Hll), _p(bl), _p(W), C.byref(chi)))
        return dict(Hpp=Hpp, bp=bp, Hll=Hll, bl=bl, W=W, chi2_robust_sum=chi.value)

    def debug_schur(self, lam, robust=True, huber_delta=HUBER_GBA, dense=False):
        S = np.empty((6 * self.K, 6 * self.K)) if dense else None
        bs = np.empty(6 * self.K); dxp = np.empty((self.K, 6)); dxl = np.empty((self.P, 3))
        it = C.c_int32(); rr = C.c_double()
        _chk(lib().ccm_ba_debug_schur(self._h, int(robust), C.c_double(huber_delta), C.c_double(lam), _p(S), _p(bs), _p(dxp), _p(dxl), C.byref(it), C.byref(rr)))
        return dict(S=S, bschur=bs, dx_pose=dxp, dx_point=dxl, pcg_iters=it.value, pcg_relres=rr.value)

    def debug_step(self, dx_pose, lam, robust=True, huber_delta=HUBER_GBA):
        """one LM trial from the given pose step x (K, 6) at damping lam, without the Schur and PCG passes: the trial state, the landmark
        step, the trial robust chi2 and the pose / landmark halves of the gain-ratio denominator (ccm_ba_debug_step)"""
        x = np.ascontiguousarray(dx_pose, np.float64).reshape(self.K, 6)
        pose = np.empty((self.K, 7)); pt = np.empty((self.P, 3)); dxl = np.empty((self.P, 3))
        chi, sp, sl = C.c_double(), C.c_double(), C.c_double()
        _chk(lib().ccm_ba_debug_step(self._h, int(robust), C.c_double(huber_delta), C.c_double(lam), _p(x), _p(pose), _p(pt), _p(dxl),
                                     C.byref(chi), C.byref(sp), C.byref(sl)))
        return dict(pose_trial=pose, pt_trial=pt, dx_point=dxl, chi2_trial=chi.value, scale_pose=sp.value, scale_point=sl.value)

    def debug_schur_blocks(self):
        """S and b_schur as the last debug_schur left them: block CSR in pose indices (rowptr (K+1,), col (nnzb,), val (nnzb,6,6)),
        fixed poses with empty rows, and b_schur (K,6)."""
        nnzb = self.info()["s_blocks_full"]
        rowptr = np.empty(self.K + 1, np.int32); col = np.empty(max(nnzb, 1), np.int32); val = np.empty((max(nnzb, 1), 6, 6))
        bs = np.empty((self.K, 6))
        _chk(lib().ccm_ba_debug_schur_blocks(self._h, _p(rowptr), _p(col), _p(val), _p(bs)))
        return dict(rowptr=rowptr, col=col[:nnzb], val=val[:nnzb], bschur=bs)

    def debug_products(self):
        """the Schur product lists (ccm_ba_debug_products): blk (nub, 2) upper blocks as (row, column) pose indices, ptr (nub+1,)
        list offsets, pairs (nprod, 2) observation pairs (e, o) as positions in the landmark-sorted observation order"""
        i = self.info()
        nub, nprod = i["s_blocks_upper"], i["schur_products"]
        blk = np.empty((max(nub, 1), 2), np.int32); ptr = np.empty(nub + 1, np.uint32); pairs = np.empty((max(nprod, 1), 2), np.int32)
        _chk(lib().ccm_ba_debug_products(self._h, _p(blk), _p(ptr), _p(pairs)))
        return dict(blk=blk[:nub], ptr=ptr.astype(np.int64), pairs=pairs[:nprod])

    def debug_schedule(self):
        """the Schur kernel's schedule (ccm_ba_debug_schedule): ntasks, grid (CTAs of its launch), task_ptr (ntasks+1,) ranges in
        sched (nub,), the upper block numbers of debug_products"""
        counts = np.zeros(2, np.int32)
        _chk(lib().ccm_ba_debug_schedule(self._h, _p(counts), None, None))
        nt, nub = int(counts[0]), self.info()["s_blocks_upper"]
        tp = np.empty(nt + 1, np.int32); sched = np.empty(max(nub, 1), np.int32)
        _chk(lib().ccm_ba_debug_schedule(self._h, None, _p(tp), _p(sched)))
        return dict(ntasks=nt, grid=int(counts[1]), task_ptr=tp, sched=sched[:nub])

    def debug_pcg2(self):
        """k_pcg2's streamed items (ccm_ba_debug_pcg2): items (nitems, 20), cta_row / cta_item (grid+1,), slab_lo (grid, 16), streamed"""
        counts = np.zeros(3, np.int64)
        _chk(lib().ccm_ba_debug_pcg2(self._h, _p(counts), None, None, None, None))
        n, g = int(counts[0]), int(counts[1])
        items = np.empty((max(n, 1), 20), np.int32); cr = np.empty(g + 1, np.int32); ci = np.empty(g + 1, np.int32)
        slo = np.empty((g, 16), np.int32)
        _chk(lib().ccm_ba_debug_pcg2(self._h, None, _p(items), _p(cr), _p(ci), _p(slo)))
        return dict(items=items[:n], cta_row=cr, cta_item=ci, slab_lo=slo, streamed=int(counts[2]))

    PATH_KEYS = ("pcg_impl", "pcg_block", "pcg_agg", "pcg_nc")

    def debug_paths(self):
        """the PCG path the handle runs: kernel, CTA size and coarse space"""
        out = np.zeros(4, np.int32)
        _chk(lib().ccm_ba_debug_paths(self._h, _p(out)))
        return {k: int(v) for k, v in zip(self.PATH_KEYS, out)}

    def debug_coarse(self):
        """the coarse level of the PCG preconditioner on the S the last debug_schur left: the assembled Galerkin matrix P^T S P
        and its inverse from the PCG set-up, both (6 nc, 6 nc)"""
        nC = 6 * self.debug_paths()["pcg_nc"]
        Ac = np.empty((nC, nC)); Ainv = np.empty((nC, nC))
        _chk(lib().ccm_ba_debug_coarse(self._h, _p(Ac), _p(Ainv)))
        return dict(Ac=Ac, Ainv=Ainv)

    def set_estimate(self, poses=None, points=None):
        """replace the estimate, keep structure and observations on the device (ccm_ba_set_estimate)"""
        ps = None if poses is None else np.ascontiguousarray(poses, np.float64)
        pt = None if points is None else np.ascontiguousarray(points, np.float64)
        _chk(lib().ccm_ba_set_estimate(self._h, _p(ps), _p(pt)))

    def pcg_cycles(self):
        """SM-clock cycles CTA 0 of the PCG kernel spent per phase (handle created with CCM_PCG_PROF=1): set-up, product, coarse, precondition, ..."""
        c = np.zeros(8, np.int64)
        _chk(lib().ccm_ba_debug_pcg_cycles(self._h, _p(c)))
        return [int(x) for x in c]

    def time_kernel(self, which, reps=5, huber_delta=HUBER_GBA, lam=1.0):
        ms = C.c_double()
        _chk(lib().ccm_ba_time_kernel(self._h, which, reps, C.c_double(huber_delta), C.c_double(lam), C.byref(ms)))
        return ms.value


def poses_from_Tcw_f32(T):
    T = np.ascontiguousarray(T, np.float32).reshape(-1, 16)
    out = np.empty((T.shape[0], 7))
    lib().ccm_pose_from_Tcw_f32(_p(T), T.shape[0], _p(out))
    return out


def poses_to_Tcw_f32(qt):
    qt = np.ascontiguousarray(qt, np.float64).reshape(-1, 7)
    out = np.empty((qt.shape[0], 4, 4), np.float32)
    lib().ccm_pose_to_Tcw_f32(_p(qt), qt.shape[0], _p(out))
    return out


def pgo_solve(p, iterations=20, lambda_init=1e-16, pcg_max_iter=0, pcg_tol=0.0, stop=None):
    arrs = dict(sim3=np.ascontiguousarray(p.sim3, np.float64), fixed=np.ascontiguousarray(p.fixed, np.uint8),
                ei=np.ascontiguousarray(p.edge_i, np.int32), ej=np.ascontiguousarray(p.edge_j, np.int32),
                meas=np.ascontiguousarray(p.meas, np.float64))
    K, E = arrs["sim3"].shape[0], arrs["ei"].shape[0]
    prob = PGOProblemC(K, E, _p(arrs["sim3"]), _p(arrs["fixed"]), _p(arrs["ei"]), _p(arrs["ej"]), _p(arrs["meas"]), int(p.fix_scale))
    out = np.empty((K, 8)); trace = np.zeros((max(iterations, 1), TRACE_COLS))
    opt = PGOOptionsC(iterations, float(lambda_init), pcg_max_iter, float(pcg_tol), _p(stop))
    res = PGOResultC(_p(out), _p(trace), trace.shape[0])
    _chk(lib().ccm_pgo_solve(C.byref(prob), C.byref(opt), C.byref(res)))
    return dict(sim3=out, trace=trace[:res.trace_len], iters_done=res.iters_done, chi2_initial=res.chi2_initial,
                chi2_final=res.chi2_final, lambda_final=res.lambda_final, t_total_ms=res.t_total_ms)


def sim3_debug_ops(u, a, b, fix_scale=False):
    """ccm_sim3_debug_ops: the device's s3_exp(u), s3_log(a), s3_mul(a, b), s3_inv(a), s3_oplus(a, u) row by row"""
    u = np.ascontiguousarray(u, np.float64).reshape(-1, 7); a = np.ascontiguousarray(a, np.float64).reshape(-1, 8)
    b = np.ascontiguousarray(b, np.float64).reshape(-1, 8)
    n = u.shape[0]
    assert a.shape[0] == n and b.shape[0] == n
    out = dict(exp=np.empty((n, 8)), log=np.empty((n, 7)), mul=np.empty((n, 8)), inv=np.empty((n, 8)), oplus=np.empty((n, 8)))
    _chk(lib().ccm_sim3_debug_ops(n, _p(u), _p(a), _p(b), int(bool(fix_scale)), *[_p(out[k]) for k in ("exp", "log", "mul", "inv", "oplus")]))
    return out


def pgo_debug_edges(meas, si, sj, free_ij, fix_scale=False):
    """ccm_pgo_debug_edges: the device's per-edge error (n,7) and Jacobians Ji, Jj (n,7,7); free_ij (n,2) != 0 marks a free side"""
    m, a, b = [np.ascontiguousarray(v, np.float64).reshape(-1, 8) for v in (meas, si, sj)]
    f = np.ascontiguousarray(free_ij, np.int32).reshape(-1, 2)
    n = m.shape[0]
    err = np.empty((n, 7)); Ji = np.empty((n, 7, 7)); Jj = np.empty((n, 7, 7))
    _chk(lib().ccm_pgo_debug_edges(n, _p(m), _p(a), _p(b), _p(f), int(bool(fix_scale)), _p(err), _p(Ji), _p(Jj)))
    return dict(err=err, Ji=Ji, Jj=Jj)


PGO_PATH_KEYS = ("pcg_block", "pcg_agg", "pcg_nc", "coarse_used")


def pgo_debug_system(p, lam, pcg_max_iter=0, pcg_tol=0.0):
    """ccm_pgo_debug_system: one linearisation at p.sim3 and one PCG solve of (H + lam I) x = b with ccm_pgo_solve's set-up.
    H is block CSR in free-vertex indices (rowptr (n+1,), col (nnzb,), H (nnzb,7,7), without lam)."""
    arrs = dict(sim3=np.ascontiguousarray(p.sim3, np.float64), fixed=np.ascontiguousarray(p.fixed, np.uint8),
                ei=np.ascontiguousarray(p.edge_i, np.int32), ej=np.ascontiguousarray(p.edge_j, np.int32),
                meas=np.ascontiguousarray(p.meas, np.float64))
    K, E = arrs["sim3"].shape[0], arrs["ei"].shape[0]
    prob = PGOProblemC(K, E, _p(arrs["sim3"]), _p(arrs["fixed"]), _p(arrs["ei"]), _p(arrs["ej"]), _p(arrs["meas"]), int(p.fix_scale))
    opt = PGOOptionsC(1, float(lam), pcg_max_iter, float(pcg_tol), None)
    n = C.c_int32(); nnzb = C.c_int64()
    f = lib().ccm_pgo_debug_system
    f.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.c_void_p, C.c_void_p] + [C.c_void_p] * 10
    _chk(f(C.byref(prob), C.byref(opt), lam, C.byref(n), C.byref(nnzb), *[None] * 10))
    n, nnzb = n.value, nnzb.value
    out = dict(vidx=np.empty(K, np.int32), rowptr=np.empty(n + 1, np.int32), col=np.empty(max(nnzb, 1), np.int32),
               H=np.empty((max(nnzb, 1), 7, 7)), b=np.empty((n, 7)), Minv=np.empty((n, 7, 7)), x=np.empty((n, 7)),
               chi2=np.empty(1), pcg=np.empty(4), paths=np.empty(4, np.int32))
    _chk(f(C.byref(prob), C.byref(opt), lam, C.byref(C.c_int32()), C.byref(C.c_int64()),
           *[_p(out[k]) for k in ("vidx", "rowptr", "col", "H", "b", "Minv", "x", "chi2", "pcg", "paths")]))
    out["col"] = out["col"][:nnzb]; out["H"] = out["H"][:nnzb]
    out.update(n=n, nnzb=nnzb, chi2=float(out["chi2"][0]), pcg_iters=int(out["pcg"][0]), pcg_relres=float(out["pcg"][1]),
               pcg_flag=int(out["pcg"][2]), pcg_nC=int(out["pcg"][3]),
               paths={k: int(v) for k, v in zip(PGO_PATH_KEYS, out["paths"])})
    return out


def hamming_matrix(A, B):
    A = np.ascontiguousarray(A, np.uint8).reshape(-1, 32); B = np.ascontiguousarray(B, np.uint8).reshape(-1, 32)
    D = np.empty((A.shape[0], B.shape[0]), np.uint16)
    _chk(lib().ccm_hamming_matrix(_p(A), A.shape[0], _p(B), B.shape[0], _p(D)))
    return D


# ---- single-vertex optimisations ---------------------------------------------------------------------------------------
class PoseOptProblemC(C.Structure):
    _fields_ = [("n", C.c_int32), ("Tcw", C.c_void_p), ("Xw", C.c_void_p), ("uv", C.c_void_p), ("inv_sigma2", C.c_void_p),
                ("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float), ("cy", C.c_float)]


class PoseOptResultC(C.Structure):
    _fields_ = [("Tcw", C.c_double * 7), ("n_inliers", C.c_int32), ("outlier", C.c_void_p)]


class Sim3OptProblemC(C.Structure):
    _fields_ = [("n", C.c_int32), ("S12", C.c_void_p), ("P1c", C.c_void_p), ("P2c", C.c_void_p), ("uv1", C.c_void_p),
                ("uv2", C.c_void_p), ("inv_sigma2_1", C.c_void_p), ("inv_sigma2_2", C.c_void_p), ("K1", C.c_float * 4),
                ("K2", C.c_float * 4), ("th2", C.c_float), ("fix_scale", C.c_int32)]


class Sim3OptResultC(C.Structure):
    _fields_ = [("S12", C.c_double * 8), ("n_inliers", C.c_int32), ("inlier", C.c_void_p)]


def _pose_probs(problems, state_key="Tcw0"):
    B = len(problems)
    probs = (PoseOptProblemC * max(B, 1))(); res = (PoseOptResultC * max(B, 1))()
    keep = []
    for b, d in enumerate(problems):
        a = dict(T=np.ascontiguousarray(d[state_key], np.float64), X=np.ascontiguousarray(d["Xw"], np.float32).reshape(-1, 3),
                 uv=np.ascontiguousarray(d["uv"], np.float32).reshape(-1, 2), w=np.ascontiguousarray(d["inv_sigma2"], np.float32))
        n = a["X"].shape[0]
        a["out"] = np.zeros(max(n, 1), np.uint8)
        keep.append(a)
        probs[b] = PoseOptProblemC(n, _p(a["T"]), _p(a["X"]), _p(a["uv"]), _p(a["w"]), *[float(v) for v in d["intr"]])
        res[b].outlier = _p(a["out"])
    return probs, res, keep


def _sim3_probs(problems, state_key="S12_0"):
    B = len(problems)
    probs = (Sim3OptProblemC * max(B, 1))(); res = (Sim3OptResultC * max(B, 1))()
    keep = []
    f32 = lambda x, c: np.ascontiguousarray(x, np.float32).reshape(-1, c) if c else np.ascontiguousarray(x, np.float32)
    for b, d in enumerate(problems):
        a = dict(S=np.ascontiguousarray(d[state_key], np.float64), P1=f32(d["P1c"], 3), P2=f32(d["P2c"], 3), u1=f32(d["uv1"], 2),
                 u2=f32(d["uv2"], 2), w1=f32(d["w1"], 0), w2=f32(d["w2"], 0))
        n = a["P1"].shape[0]
        a["inl"] = np.zeros(max(n, 1), np.uint8)
        keep.append(a)
        probs[b] = Sim3OptProblemC(n, _p(a["S"]), _p(a["P1"]), _p(a["P2"]), _p(a["u1"]), _p(a["u2"]), _p(a["w1"]), _p(a["w2"]),
                                   (C.c_float * 4)(*[float(v) for v in d["K1"]]), (C.c_float * 4)(*[float(v) for v in d["K2"]]),
                                   float(d["th2"]), int(bool(d["fix_scale"])))
        res[b].inlier = _p(a["inl"])
    return probs, res, keep


SINGLE_TRACE_CALL = 7 + 10 * 7     # CCM_SINGLE_TRACE_HEAD + CCM_SINGLE_TRACE_ITERS * CCM_SINGLE_TRACE_COLS
SINGLE_TRACE_CALLS = {"pose": 4, "sim3": 2}


def pose_optimize(problems, trace=False):
    """Optimizer::PoseOptimizationClient for a batch of frames.  problems: list of dict(Tcw0, Xw, uv, inv_sigma2, intr)
    (ccm_slam_b200.synth.make_pose_opt layout).  Returns a list of (Tcw (7,), outlier (n,) u8, n_inliers); with trace=True
    (ccm_pose_optimize_traced, test only) each tuple also carries the LM trace (4, SINGLE_TRACE_CALL)."""
    B = len(problems)
    probs, res, keep = _pose_probs(problems)
    if trace:
        tr = np.empty((max(B, 1), SINGLE_TRACE_CALLS["pose"], SINGLE_TRACE_CALL))
        _chk(lib().ccm_pose_optimize_traced(probs, B, res, _p(tr)))
    else:
        _chk(lib().ccm_pose_optimize(probs, B, res))
    return [(np.array(res[b].Tcw[:]), keep[b]["out"][:keep[b]["X"].shape[0]], int(res[b].n_inliers)) + ((tr[b],) if trace else ())
            for b in range(B)]


def sim3_optimize(problems, trace=False):
    """Optimizer::OptimizeSim3 for a batch of keyframe pairs.  problems: list of dict(S12_0, P1c, P2c, uv1, uv2, w1, w2, K1, K2,
    th2, fix_scale) (synth.make_sim3_opt layout).  Returns a list of (S12 (8,), inlier (n,) u8, n_inliers); with trace=True
    (ccm_sim3_optimize_traced, test only) each tuple also carries the LM trace (2, SINGLE_TRACE_CALL)."""
    B = len(problems)
    probs, res, keep = _sim3_probs(problems)
    if trace:
        tr = np.empty((max(B, 1), SINGLE_TRACE_CALLS["sim3"], SINGLE_TRACE_CALL))
        _chk(lib().ccm_sim3_optimize_traced(probs, B, res, _p(tr)))
    else:
        _chk(lib().ccm_sim3_optimize(probs, B, res))
    return [(np.array(res[b].S12[:]), keep[b]["inl"][:keep[b]["P1"].shape[0]], int(res[b].n_inliers)) + ((tr[b],) if trace else ())
            for b in range(B)]


def single_debug_system(kind, problems, states, active, robust, delta, lam):
    """ccm_pose_debug_system (kind "pose", D = 6) / ccm_sim3_debug_system ("sim3", D = 7): per problem b, at states[b], with the
    per-edge masks active[b], robust[b] (n / 2n entries), Huber delta[b] and lambda lam[b]: one system build and one damped solve
    with the optimiser's device functions.  Returns per problem dict(err (E,2), J (E,2,D), H (D,D), b (D,), chi2, x (D,), solved)."""
    D, per = (6, 1) if kind == "pose" else (7, 2)
    key = "Tcw0" if kind == "pose" else "S12_0"
    probs_l = [{"th2": 0.0, **d, key: np.asarray(s, np.float64)} for d, s in zip(problems, states)]   # th2 is not read here
    probs, _, keep = (_pose_probs if kind == "pose" else _sim3_probs)(probs_l)
    B = len(problems)
    ne = [per * (k["X"] if kind == "pose" else k["P1"]).shape[0] for k in keep]
    tot = sum(ne)
    act = np.ascontiguousarray(np.concatenate([np.asarray(a, np.uint8).ravel() for a in active]) if B else np.zeros(0, np.uint8), np.uint8)
    rob = np.ascontiguousarray(np.concatenate([np.asarray(a, np.uint8).ravel() for a in robust]) if B else np.zeros(0, np.uint8), np.uint8)
    assert act.size == tot and rob.size == tot
    dl = np.ascontiguousarray(np.stack([np.asarray(delta, np.float64), np.asarray(lam, np.float64)], 1) if B else np.zeros((1, 2)))
    err = np.empty((max(tot, 1), 2)); J = np.empty((max(tot, 1), 2, D)); ns = D * D + 2 * D + 1
    sys_ = np.empty((max(B, 1), ns)); sol = np.empty(max(B, 1), np.int32)
    f = lib().ccm_pose_debug_system if kind == "pose" else lib().ccm_sim3_debug_system
    _chk(f(probs, B, _p(act), _p(rob), _p(dl), _p(err), _p(J), _p(sys_), _p(sol)))
    out, o = [], 0
    for b in range(B):
        s = sys_[b]
        out.append(dict(err=err[o:o + ne[b]].copy(), J=J[o:o + ne[b]].copy(), H=s[:D * D].reshape(D, D).copy(), b=s[D * D:D * D + D].copy(),
                        chi2=float(s[D * D + D]), x=s[D * D + D + 1:].copy(), solved=bool(sol[b])))
        o += ne[b]
    return out


def _map_update_args(sc):
    """flat map view (ccm_slam_b200.synth.make_map_update layout) -> contiguous arrays + outputs for ccm_gba_map_update / its mirrors"""
    K = len(sc["kf_parent"]); P = len(sc["mp_state"])
    a = dict(parent=np.ascontiguousarray(sc["kf_parent"], np.int32), opt=np.ascontiguousarray(sc["kf_optimized"], np.uint8),
             Tcw=np.ascontiguousarray(sc["kf_Tcw"], np.float32).reshape(K, 16), gba=np.array(sc["kf_TcwGBA"], np.float32).reshape(K, 16),
             vis=np.zeros(max(K, 1), np.uint8), state=np.ascontiguousarray(sc["mp_state"], np.uint8), ref=np.ascontiguousarray(sc["mp_ref"], np.int32),
             pos=np.ascontiguousarray(sc["mp_pos"], np.float32).reshape(P, 3), pgba=np.ascontiguousarray(sc["mp_pos_gba"], np.float32).reshape(P, 3),
             out=np.zeros((max(P, 1), 3), np.float32), corr=np.zeros(max(P, 1), np.uint8))
    argv = (K, _p(a["parent"]), _p(a["opt"]), _p(a["Tcw"]), _p(a["gba"]), _p(a["vis"]), P, _p(a["state"]), _p(a["ref"]), _p(a["pos"]), _p(a["pgba"]),
            _p(a["out"]), _p(a["corr"]))
    return a, argv, K, P


def _map_update_result(a, K, P):
    return dict(kf_TcwGBA=a["gba"].reshape(K, 4, 4), kf_visited=a["vis"][:K], mp_pos=a["out"][:P], mp_corrected=a["corr"][:P])


def gba_map_update(sc):
    """The map update after a global BA (Map::RunGBA, S/Map.cpp:1441-1570 = MapMerger::RunGBA, S/MapMerger.cpp:637-753) on a flat view
    of the map: dict(kf_parent, kf_optimized, kf_Tcw (K,4,4) f32, kf_TcwGBA, mp_state, mp_ref, mp_pos, mp_pos_gba), see include/ccm_b200.h.
    Returns dict(kf_TcwGBA, kf_visited, mp_pos, mp_corrected).  Keyframe pass on the host, point pass on the GPU."""
    a, argv, K, P = _map_update_args(sc)
    _chk(lib().ccm_gba_map_update(*argv))
    return _map_update_result(a, K, P)


def normal_depth(sc, host=False):
    """MapPoint::UpdateNormalAndDepth (cslam/src/MapPoint.cpp:779-823) for a batch of points, see include/ccm_b200.h.  sc: dict(kf_centre
    (K,3) f32, kf_bad (K,) u8, mp_pos (P,3) f32, obs_ptr (P+1,) i64, obs_kf (E,) i32, mp_ref (P,) i32, mp_scale_ref, mp_scale_last (P,) f32).
    Returns dict(normal (P,3), max_dist, min_dist, status).  host=False: ccm_normal_depth on the GPU; host=True: ccm_normal_depth_host."""
    K = len(sc["kf_bad"]); P = len(sc["mp_ref"])
    a = dict(c=np.ascontiguousarray(sc["kf_centre"], np.float32).reshape(K, 3), bad=np.ascontiguousarray(sc["kf_bad"], np.uint8),
             pos=np.ascontiguousarray(sc["mp_pos"], np.float32).reshape(P, 3), ptr=np.ascontiguousarray(sc["obs_ptr"], np.int64),
             obs=np.ascontiguousarray(sc["obs_kf"], np.int32), ref=np.ascontiguousarray(sc["mp_ref"], np.int32),
             sr=np.ascontiguousarray(sc["mp_scale_ref"], np.float32), sl=np.ascontiguousarray(sc["mp_scale_last"], np.float32))
    out = dict(normal=np.zeros((P, 3), np.float32), max_dist=np.zeros(P, np.float32), min_dist=np.zeros(P, np.float32),
               status=np.zeros(P, np.uint8))
    fn = lib().ccm_normal_depth_host if host else lib().ccm_normal_depth
    _chk(fn(K, _p(a["c"]), _p(a["bad"]), P, _p(a["pos"]), _p(a["ptr"]), _p(a["obs"]), _p(a["ref"]), _p(a["sr"]), _p(a["sl"]),
            _p(out["normal"]), _p(out["max_dist"]), _p(out["min_dist"]), _p(out["status"])))
    return out



def distinctive_descriptors(sc, host=False):
    """MapPoint::ComputeDistinctiveDescriptors (cslam/src/MapPoint.cpp:929-994) for a batch of points, see include/ccm_b200.h.  sc: dict(
    kf_bad (K,) u8, obs_ptr (P+1,) i64, obs_kf (E,) i32, obs_desc (E,32) u8), as synth.make_distinctive builds it.  Returns dict(best (P,)
    i32: position of the chosen observer in the point's list, -1 untouched; best_median (P,) i32; desc (P,32) u8).  host=False:
    ccm_distinctive_descriptors on the GPU; host=True: ccm_distinctive_descriptors_host."""
    K = len(sc["kf_bad"]); P = len(sc["obs_ptr"]) - 1
    a = dict(bad=np.ascontiguousarray(sc["kf_bad"], np.uint8), ptr=np.ascontiguousarray(sc["obs_ptr"], np.int64),
             obs=np.ascontiguousarray(sc["obs_kf"], np.int32), desc=np.ascontiguousarray(sc["obs_desc"], np.uint8).reshape(-1, 32))
    out = dict(best=np.zeros(P, np.int32), best_median=np.zeros(P, np.int32), desc=np.zeros((P, 32), np.uint8))
    fn = lib().ccm_distinctive_descriptors_host if host else lib().ccm_distinctive_descriptors
    _chk(fn(K, _p(a["bad"]), P, _p(a["ptr"]), _p(a["obs"]), _p(a["desc"]), _p(out["best"]), _p(out["best_median"]), _p(out["desc"])))
    return out


def covisibility_batch(sc, batch=None):
    """The batch arrays of ccm_covisibility for the keyframe rows `batch` (None: sc["batch"]) of a scene as synth.make_covisibility
    builds it: batch (B,) i32, kf_mp_ptr (B+1,) i64, kf_mp i32 (each row's mvpMapPoints in index order, -1 null)."""
    batch = np.ascontiguousarray(sc["batch"] if batch is None else batch, np.int32)
    mptr = np.asarray(sc["mvp_ptr"], np.int64)
    n = mptr[batch + 1] - mptr[batch]
    ptr = np.zeros(len(batch) + 1, np.int64); ptr[1:] = np.cumsum(n)
    idx = np.repeat(mptr[batch] - ptr[:-1], n) + np.arange(ptr[-1])
    return batch, ptr, np.ascontiguousarray(np.asarray(sc["mvp"], np.int32)[idx])


def covisibility(sc, th=15, host=False, capacity=None, batch=None):
    """KeyFrame::UpdateConnections' weights and ordered connections (cslam/src/KeyFrame.cpp:629-711) for a batch of keyframes, see
    include/ccm_b200.h.  sc: dict(kf_id (K,) u64, kf_rank (K,) u32, mvp_ptr (K+1,) i64, mvp, mp_bad (P,) u8, obs_ptr (P+1,) i64, obs_kf,
    batch), as synth.make_covisibility builds it.  Returns dict(conn_ptr (B+1,) i64, conn_kf, conn_w: KFcounter by ascending rank;
    n_sel (B,), sel_kf, sel_w: the ordered selection in the first n_sel slots of each range; status (B,) u8).  host=False:
    ccm_covisibility on the GPU; host=True: ccm_covisibility_host.  capacity None: a guess, then the exact total if refused."""
    b, mptr, mp = covisibility_batch(sc, batch)
    B = len(b)
    a = [np.ascontiguousarray(sc[k], t) for k, t in (("kf_id", np.uint64), ("kf_rank", np.uint32), ("mp_bad", np.uint8),
                                                     ("obs_ptr", np.int64), ("obs_kf", np.int32))]
    fn = lib().ccm_covisibility_host if host else lib().ccm_covisibility
    total = np.zeros(1, np.int64)
    cap = int(capacity) if capacity is not None else min(int(mptr[-1]) * 32, 64 * B + 4096)
    while True:
        out = dict(conn_ptr=np.zeros(B + 1, np.int64), conn_kf=np.zeros(max(cap, 1), np.int32), conn_w=np.zeros(max(cap, 1), np.int32),
                   n_sel=np.zeros(B, np.int32), sel_kf=np.zeros(max(cap, 1), np.int32), sel_w=np.zeros(max(cap, 1), np.int32),
                   status=np.zeros(B, np.uint8))
        rc = fn(len(a[0]), _p(a[0]), _p(a[1]), B, _p(b), _p(mptr), _p(mp), len(a[2]), _p(a[2]), _p(a[3]), _p(a[4]), int(th), C.c_int64(cap),
                _p(out["conn_ptr"]), _p(out["conn_kf"]), _p(out["conn_w"]), _p(out["n_sel"]), _p(out["sel_kf"]), _p(out["sel_w"]),
                _p(out["status"]), _p(total))
        if rc != 0 and capacity is None and total[0] > cap:
            cap = int(total[0])
            continue
        _chk(rc)
        break
    T = int(total[0])
    for k in ("conn_kf", "conn_w", "sel_kf", "sel_w"):
        out[k] = out[k][:T]
    return out

SIM3_CORRECTION_IN = (("kf_centre", np.float32), ("kf_bad", np.uint8), ("entry_kf", np.int32), ("entry_Siw_new", np.float64),
                      ("entry_Siw_old", np.float64), ("slot_ptr", np.int64), ("slot_mp", np.int32), ("mp_pos", np.float32),
                      ("mp_skip", np.uint8), ("obs_ptr", np.int64), ("obs_kf", np.int32), ("mp_ref", np.int32), ("mp_scale_ref", np.float32),
                      ("mp_scale_last", np.float32))


def sim3_correction_out(n_e, n_mp):
    """zeroed outputs of ccm_sim3_correction for n_e entries and n_mp points"""
    return dict(entry_Tcw=np.zeros((n_e, 4, 4), np.float32), entry_centre=np.zeros((n_e, 3), np.float32), mp_entry=np.zeros(n_mp, np.int32),
                mp_pos=np.zeros((n_mp, 3), np.float32), normal=np.zeros((n_mp, 3), np.float32), max_dist=np.zeros(n_mp, np.float32),
                min_dist=np.zeros(n_mp, np.float32), status=np.zeros(n_mp, np.uint8))


def sim3_correction_args(sc, out):
    """(argument tuple of ccm_sim3_correction, arrays it points into) for a scene as synth.make_sim3_correction builds it"""
    a = {k: np.ascontiguousarray(sc[k], t) for k, t in SIM3_CORRECTION_IN}
    K, E, P = len(a["kf_bad"]), len(a["entry_kf"]), len(a["mp_skip"])
    argv = (K, _p(a["kf_centre"]), _p(a["kf_bad"]), E, _p(a["entry_kf"]), _p(a["entry_Siw_new"]), _p(a["entry_Siw_old"]), _p(a["slot_ptr"]),
            _p(a["slot_mp"]), P, _p(a["mp_pos"]), _p(a["mp_skip"]), _p(a["obs_ptr"]), _p(a["obs_kf"]), _p(a["mp_ref"]), _p(a["mp_scale_ref"]),
            _p(a["mp_scale_last"]), _p(out["entry_Tcw"]), _p(out["entry_centre"]), _p(out["mp_entry"]), _p(out["mp_pos"]), _p(out["normal"]),
            _p(out["max_dist"]), _p(out["min_dist"]), _p(out["status"]))
    return argv, a


def sim3_correction(sc, host=False, out=None):
    """The Sim3 correction pass of LoopFinder::CorrectLoop / MapMerger::MergeMaps (cslam/src/LoopFinder.cpp:568-613,
    cslam/src/MapMerger.cpp:349-395), see include/ccm_b200.h.  sc: dict(kf_centre (K,3) f32, kf_bad (K,) u8, entry_kf (E,) i32,
    entry_Siw_new / entry_Siw_old (E,8) f64, slot_ptr (E+1,) i64, slot_mp i32, mp_pos (P,3) f32, mp_skip (P,) u8, obs_ptr (P+1,) i64,
    obs_kf i32, mp_ref (P,) i32, mp_scale_ref / mp_scale_last (P,) f32), as synth.make_sim3_correction builds it.  Returns dict(entry_Tcw
    (E,4,4) f32, entry_centre (E,3), mp_entry (P,) i32, mp_pos (P,3), normal (P,3), max_dist, min_dist, status).  host=False:
    ccm_sim3_correction on the GPU; host=True: ccm_sim3_correction_host.  out: preallocated outputs (sim3_correction_out)."""
    out = sim3_correction_out(len(sc["entry_kf"]), len(sc["mp_skip"])) if out is None else out
    argv, _keep = sim3_correction_args(sc, out)
    fn = lib().ccm_sim3_correction_host if host else lib().ccm_sim3_correction
    _chk(fn(*argv))
    return out


KEYFRAME_CULLING_IN = (("kf_bad", np.uint8), ("cand_kf", np.int32), ("cand_not_erase", np.uint8), ("slot_ptr", np.int64),
                       ("slot_mp", np.int32), ("slot_octave", np.int32), ("mp_bad", np.uint8), ("mp_nobs", np.int32), ("mp_ref", np.int32),
                       ("obs_ptr", np.int64), ("obs_kf", np.int32), ("obs_octave", np.int32))


def keyframe_culling_out(n_c):
    """zeroed outputs of ccm_keyframe_culling for n_c candidates"""
    return dict(cull=np.zeros(n_c, np.uint8), n_mps=np.zeros(n_c, np.int32), n_red=np.zeros(n_c, np.int32), n_settled=np.zeros(1, np.int32))


def keyframe_culling_args(sc, out):
    """(argument tuple of ccm_keyframe_culling, arrays it points into) for the flat arrays of a scene as
    synth.make_keyframe_culling_scene builds it (th_obs and red_thres from the scene, 3 and 0.98 when absent)"""
    a = {k: np.ascontiguousarray(sc[k], t) for k, t in KEYFRAME_CULLING_IN}
    K, Cn, P = len(a["kf_bad"]), len(a["cand_kf"]), len(a["mp_bad"])
    argv = (K, _p(a["kf_bad"]), Cn, _p(a["cand_kf"]), _p(a["cand_not_erase"]), _p(a["slot_ptr"]), _p(a["slot_mp"]), _p(a["slot_octave"]), P,
            _p(a["mp_bad"]), _p(a["mp_nobs"]), _p(a["mp_ref"]), _p(a["obs_ptr"]), _p(a["obs_kf"]), _p(a["obs_octave"]), int(sc.get("th_obs", 3)),
            C.c_double(float(sc.get("red_thres", 0.98))), _p(out["cull"]), _p(out["n_mps"]), _p(out["n_red"]), _p(out["n_settled"]))
    return argv, a


def keyframe_culling(sc, host=False, out=None):
    """The redundancy test of LocalMapping::KeyFrameCullingV3 (cslam/src/Mapping.cpp:771-863) for every candidate, earlier culls
    included, see include/ccm_b200.h.  sc: dict(kf_bad (K,) u8, cand_kf (C,) i32, cand_not_erase (C,) u8, slot_ptr (C+1,) i64, slot_mp,
    slot_octave i32, mp_bad (P,) u8, mp_nobs (P,) i32, mp_ref (P,) i32, obs_ptr (P+1,) i64, obs_kf, obs_octave i32, th_obs, red_thres),
    as synth.make_keyframe_culling_scene builds it.  Returns dict(cull (C,) u8, n_mps (C,) i32, n_red (C,) i32, n_settled int).
    host=False: ccm_keyframe_culling on the GPU; host=True: ccm_keyframe_culling_host.  out: preallocated outputs (keyframe_culling_out)."""
    out = keyframe_culling_out(len(sc["cand_kf"])) if out is None else out
    argv, _keep = keyframe_culling_args(sc, out)
    fn = lib().ccm_keyframe_culling_host if host else lib().ccm_keyframe_culling
    _chk(fn(*argv))
    return dict(cull=out["cull"], n_mps=out["n_mps"], n_red=out["n_red"], n_settled=int(out["n_settled"][0]))


class NewPtsViewC(C.Structure):
    _fields_ = [("v", TriViewC), ("Tcw", C.c_float * 12), ("Ow", C.c_float * 3), ("level_sigma2", C.c_void_p),
                ("scale_factors", C.c_void_p), ("nlevels", C.c_int32), ("scale_factor", C.c_float)]


class NewPtsNeighbourC(C.Structure):
    _fields_ = [("view", NewPtsViewC), ("F12", C.c_float * 9), ("ex", C.c_float), ("ey", C.c_float)]


NEW_POINT_DTYPE = np.dtype([("nb", np.int32), ("idx1", np.int32), ("idx2", np.int32), ("x3D", np.float32, 3)])
NEWPTS_VERDICTS = ("none", "accepted", "parallax", "w_zero", "depth1", "depth2", "reproj1", "reproj2", "dist_zero", "scale", "claimed")


def new_points_structs(cur, neighbours, keep):
    """The C structs of ccm_new_map_points for view dicts as synth_match.make_new_points_scene builds them; `keep` collects what
    must outlive the call.  A view: desc (n,32) u8, has_mp, kp_xy (n,2), octave, angle, node (n,) vocabulary node of each feature,
    intr (fx, fy, cx, cy), Tcw (3,4), Ow, level_sigma2, scale_factors, scale_factor; a neighbour adds F12 (3,3), ex, ey."""
    def view(v):
        n = len(v["octave"])
        a = dict(desc=np.ascontiguousarray(v["desc"], np.uint8), has=np.ascontiguousarray(v["has_mp"], np.uint8),
                 xy=np.ascontiguousarray(v["kp_xy"], np.float32), oc=np.ascontiguousarray(v["octave"], np.int32),
                 an=np.ascontiguousarray(v["angle"], np.float32), ls=np.ascontiguousarray(v["level_sigma2"], np.float32),
                 sf=np.ascontiguousarray(v["scale_factors"], np.float32))
        node = np.asarray(v["node"])
        ids, counts = np.unique(node, return_counts=True)
        a["node_id"] = ids.astype(np.uint32)
        a["node_ptr"] = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
        a["feat"] = np.argsort(node, kind="stable").astype(np.uint32)
        for k in ("node_id", "node_ptr", "feat"):          # a test may hand in a malformed FeatureVector
            if "fv_" + k in v:
                a[k] = np.ascontiguousarray(v["fv_" + k], a[k].dtype)
        fv = FeatureVectorC(len(a["node_id"]), _p(a["node_id"]), _p(a["node_ptr"]), _p(a["feat"]))
        keep.extend([a, fv])
        fx, fy, cx, cy = (float(x) for x in v["intr"])
        tv = TriViewC(_p(a["desc"]), n, _p(a["has"]), _p(a["xy"]), _p(a["oc"]), _p(a["an"]), C.pointer(fv), fx, fy, cx, cy)
        T = (C.c_float * 12)(*np.asarray(v["Tcw"], np.float32).reshape(12))
        O = (C.c_float * 3)(*np.asarray(v["Ow"], np.float32).reshape(3))
        return NewPtsViewC(tv, T, O, _p(a["ls"]), _p(a["sf"]), len(a["ls"]), float(v["scale_factor"]))
    c = view(cur)
    nbs = (NewPtsNeighbourC * max(len(neighbours), 1))()
    for i, v in enumerate(neighbours):
        nbs[i] = NewPtsNeighbourC(view(v), (C.c_float * 9)(*np.asarray(v["F12"], np.float32).reshape(9)), float(v["ex"]), float(v["ey"]))
    return c, nbs


def new_map_points(cur, neighbours, want_debug=False, host=False, capacity=None, fn=None):
    """LocalMapping::CreateNewMapPoints (cslam/src/Mapping.cpp:284-469) for `cur` and all `neighbours` in one call, see
    include/ccm_b200.h.  Returns the new points as a structured array (nb, idx1, idx2, x3D) in the reference's creation order; with
    want_debug also best2 and verdict, each (len(neighbours), n).  host=False: ccm_new_map_points on the GPU; host=True:
    ccm_new_map_points_host.  capacity None: room for every (neighbour, feature) pair."""
    keep = []
    c, nbs = new_points_structs(cur, neighbours, keep)
    n, B = len(cur["octave"]), len(neighbours)
    cap = n * B if capacity is None else int(capacity)
    out = np.zeros(max(cap, 1), NEW_POINT_DTYPE)
    n_out = C.c_int32(-1)
    best2 = np.full((B, n), -2, np.int32) if want_debug else None
    verdict = np.full((B, n), 255, np.uint8) if want_debug else None
    fn = fn or (lib().ccm_new_map_points_host if host else lib().ccm_new_map_points)
    rc = fn(C.byref(c), nbs, B, _p(out), cap, C.byref(n_out), _p(best2), _p(verdict))
    if rc != 0:
        e = CCMError(rc, lib().ccm_last_error().decode())
        e.needed = n_out.value
        raise e
    pts = out[:n_out.value].copy()
    return (pts, best2, verdict) if want_debug else pts


class FeatureGridC(C.Structure):
    _fields_ = [("n", C.c_int32), ("desc", C.c_void_p), ("kp_xy", C.c_void_p), ("octave", C.c_void_p), ("angle", C.c_void_p),
                ("min_x", C.c_float), ("min_y", C.c_float), ("max_x", C.c_float), ("max_y", C.c_float),
                ("grid_w_inv", C.c_float), ("grid_h_inv", C.c_float), ("grid_cols", C.c_int32), ("grid_rows", C.c_int32)]


def grid_struct(g, keep):
    """ccm_feature_grid from dict(desc, kp_xy, octave, angle, bounds=(mnMinX, mnMinY, mnMaxX, mnMaxY), cols, rows)"""
    a = dict(desc=np.ascontiguousarray(g["desc"], np.uint8), xy=np.ascontiguousarray(g["kp_xy"], np.float32),
             oc=np.ascontiguousarray(g["octave"], np.int32), an=np.ascontiguousarray(g["angle"], np.float32))
    keep.append(a)
    x0, y0, x1, y1 = [np.float32(v) for v in g["bounds"]]
    wi = np.float32(g["cols"]) / np.float32(x1 - x0)   # mfGridElementWidthInv  (S/Frame.cpp:86)
    hi = np.float32(g["rows"]) / np.float32(y1 - y0)   # mfGridElementHeightInv (S/Frame.cpp:87)
    return FeatureGridC(a["desc"].shape[0], _p(a["desc"]), _p(a["xy"]), _p(a["oc"]), _p(a["an"]), x0, y0, x1, y1, wi, hi,
                        int(g["cols"]), int(g["rows"]))


class FuseKfC(C.Structure):
    _fields_ = [("grid", FeatureGridC), ("Tcw", C.c_float * 12), ("Ow", C.c_float * 3), ("fx", C.c_float), ("fy", C.c_float),
                ("cx", C.c_float), ("cy", C.c_float), ("scale_factors", C.c_void_p), ("inv_level_sigma2", C.c_void_p),
                ("nlevels", C.c_int32), ("log_scale_factor", C.c_float)]


class FusePointsC(C.Structure):
    _fields_ = [("n", C.c_int32), ("pos", C.c_void_p), ("normal", C.c_void_p), ("max_distance", C.c_void_p),
                ("min_distance", C.c_void_p), ("desc", C.c_void_p), ("skip", C.c_void_p)]


def fuse_structs(sc, keep):
    """The C structs of ccm_fuse_neighbours for a scene as synth_match.make_fuse_scene builds it; `keep` collects what must outlive
    the call.  A keyframe: a grid dict (desc, kp_xy, octave, angle, bounds, cols, rows) plus Tcw (3,4), Ow, intr (fx, fy, cx, cy),
    scale_factors, inv_level_sigma2, log_scale_factor.  sc: cur, targets (distinct keyframes), points dict(pos (P,3), normal (P,3),
    max_d, min_d, desc (P,32), skip), cur_point (n,) and cand rows."""
    cur = fuse_kf_struct(sc["cur"], keep)
    T = len(sc["targets"])
    tg = (FuseKfC * max(T, 1))()
    for i, k in enumerate(sc["targets"]):
        tg[i] = fuse_kf_struct(k, keep)
    a = dict(cp=np.ascontiguousarray(sc["cur_point"], np.int32), cand=np.ascontiguousarray(sc["cand"], np.int32))
    keep += [a, tg]
    return cur, tg, T, fuse_points_struct(sc["points"], keep), a["cp"], a["cand"]


def fuse_kf_struct(k, keep, Tcw="Tcw", Ow="Ow"):
    """ccm_fuse_kf of one keyframe dict (see fuse_structs); Tcw / Ow name the keys the camera is read from"""
    a = dict(sf=np.ascontiguousarray(k["scale_factors"], np.float32), il=np.ascontiguousarray(k["inv_level_sigma2"], np.float32))
    keep.append(a)
    fx, fy, cx, cy = (float(x) for x in k["intr"])
    return FuseKfC(grid_struct(k, keep), (C.c_float * 12)(*np.asarray(k[Tcw], np.float32).reshape(12)),
                   (C.c_float * 3)(*np.asarray(k[Ow], np.float32).reshape(3)), fx, fy, cx, cy, _p(a["sf"]), _p(a["il"]),
                   len(a["sf"]), float(k["log_scale_factor"]))


def fuse_points_struct(p, keep, skip="skip"):
    """ccm_fuse_points of dict(pos (P,3), normal (P,3), max_d, min_d, desc (P,32), skip); `skip` names the key of the skip flags"""
    a = dict(pos=np.ascontiguousarray(p["pos"], np.float32).reshape(-1, 3), nrm=np.ascontiguousarray(p["normal"], np.float32).reshape(-1, 3),
             mx=np.ascontiguousarray(p["max_d"], np.float32), mn=np.ascontiguousarray(p["min_d"], np.float32),
             desc=np.ascontiguousarray(p["desc"], np.uint8).reshape(-1, 32), skip=np.ascontiguousarray(p[skip], np.uint8))
    keep.append(a)
    return FusePointsC(len(a["mx"]), _p(a["pos"]), _p(a["nrm"]), _p(a["mx"]), _p(a["mn"]), _p(a["desc"]), _p(a["skip"]))


def fuse_neighbours(sc, host=False, fn=None):
    """The searches of LocalMapping::SearchInNeighbors (cslam/src/Mapping.cpp:471-547) in one call, see include/ccm_b200.h.
    Returns (fwd (T, n) i32: keypoint of target t for the current keyframe's slot i or -1; bwd (C,) i32: keypoint of the current
    keyframe for candidate c or -1; the number of pairs whose PredictScale level was settled with the host's logf).
    host=False: ccm_fuse_neighbours on the GPU; host=True: ccm_fuse_neighbours_host."""
    keep = []
    cur, tg, T, pts, cp, cand = fuse_structs(sc, keep)
    n = len(cp)
    fwd = np.full((T, n), -3, np.int32)
    bwd = np.full(len(cand), -3, np.int32)
    settled = C.c_int32(-1)
    fn = fn or (lib().ccm_fuse_neighbours_host if host else lib().ccm_fuse_neighbours)
    _chk(fn(C.byref(cur), tg, T, C.byref(pts), _p(cp), _p(cand), len(cand), _p(fwd), _p(bwd), C.byref(settled)))
    return fwd, bwd, settled.value


def search_and_fuse_structs(sc, keep, Tcw="Tcw", Ow="Ow", skip="skip"):
    """The C structs of ccm_search_and_fuse for a scene as synth_match.make_search_and_fuse_scene builds it -> (kfs, n_kf, pts).
    sc: kfs (keyframe dicts as fuse_structs takes them, Tcw / Ow the split of the corrected Scw), points (the loop points, skip = isBad())."""
    K = len(sc["kfs"])
    kfs = (FuseKfC * max(K, 1))()
    for i, k in enumerate(sc["kfs"]):
        kfs[i] = fuse_kf_struct(k, keep, Tcw, Ow)
    keep.append(kfs)
    return kfs, K, fuse_points_struct(sc["points"], keep, skip)


def search_and_fuse(sc, host=False, fn=None):
    """The searches of LoopFinder / MapMerger::SearchAndFuse (cslam/src/LoopFinder.cpp:709-734, MapMerger.cpp:574-598) for every
    corrected keyframe in one call, see include/ccm_b200.h.  Returns (best (K, P) i32: keypoint of keyframe k that loop point i lands on,
    or -1; the number of pairs whose PredictScale level was settled with the host's logf).
    host=False: ccm_search_and_fuse on the GPU; host=True: ccm_search_and_fuse_host."""
    keep = []
    kfs, K, pts = search_and_fuse_structs(sc, keep)
    best = np.full((K, pts.n), -3, np.int32)
    settled = C.c_int32(-1)
    fn = fn or (lib().ccm_search_and_fuse_host if host else lib().ccm_search_and_fuse)
    _chk(fn(kfs, K, C.byref(pts), _p(best), C.byref(settled)))
    return best, settled.value


class MapMirror:
    """Persistent flat mirror of the map for the global BA (ccm_mirror_*, include/ccm_b200.h; SURVEY.md §8(f) rank 1): told about
    changes as they happen, hands out the ccm_ba_problem MapFusionGBA's flattening (S/Optimizer.cpp:658-787) would build."""

    def __init__(self):
        L = lib()
        L.ccm_mirror_rebuilds.restype = C.c_longlong
        for f in ("ccm_mirror_set_keyframe", "ccm_mirror_erase_keyframe", "ccm_mirror_set_point", "ccm_mirror_erase_point"):
            getattr(L, f).argtypes = None
        L.ccm_mirror_set_observation.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_float, C.c_float, C.c_float]
        L.ccm_mirror_erase_observation.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64]
        L.ccm_mirror_destroy.argtypes = [C.c_void_p]
        L.ccm_mirror_rebuilds.argtypes = [C.c_void_p]
        self._h = C.c_void_p()
        _chk(L.ccm_mirror_create(C.byref(self._h)))

    def close(self):
        if self._h:
            lib().ccm_mirror_destroy(self._h); self._h = C.c_void_p()

    def set_keyframe(self, uid, Tcw, intr=None, bad=False):
        T = np.ascontiguousarray(Tcw, np.float32).reshape(16)
        k = None if intr is None else np.ascontiguousarray(intr, np.float32)
        _chk(lib().ccm_mirror_set_keyframe(self._h, C.c_uint64(uid), _p(T), _p(k), int(bad)))

    def erase_keyframe(self, uid):
        _chk(lib().ccm_mirror_erase_keyframe(self._h, C.c_uint64(uid)))

    def set_point(self, uid, pos, bad=False):
        x = np.ascontiguousarray(pos, np.float32).reshape(3)
        _chk(lib().ccm_mirror_set_point(self._h, C.c_uint64(uid), _p(x), int(bad)))

    def erase_point(self, uid):
        _chk(lib().ccm_mirror_erase_point(self._h, C.c_uint64(uid)))

    def set_observation(self, kf_uid, mp_uid, u, v, inv_sigma2):
        _chk(lib().ccm_mirror_set_observation(self._h, kf_uid, mp_uid, float(u), float(v), float(inv_sigma2)))

    def erase_observation(self, kf_uid, mp_uid):
        _chk(lib().ccm_mirror_erase_observation(self._h, kf_uid, mp_uid))

    def rebuilds(self):
        return lib().ccm_mirror_rebuilds(self._h)

    def set_min_edges(self, n):
        """2 = MapFusionGBA's point rule (default), 1 = BundleAdjustmentClient's"""
        lib().ccm_mirror_set_min_edges.argtypes = [C.c_void_p, C.c_int32]
        _chk(lib().ccm_mirror_set_min_edges(self._h, int(n)))

    def problem(self, max_kf_uid, fixed_uids):
        """-> (BAProblemC over the mirror's own arrays (valid until the next call on the mirror), numpy copies of every array,
        kf_uid_of_row, mp_uid_of_row)"""
        fx = np.ascontiguousarray(fixed_uids, np.uint64)
        prob = BAProblemC(); ku = C.c_void_p(); mu = C.c_void_p()
        _chk(lib().ccm_mirror_ba_problem(self._h, C.c_uint64(max_kf_uid), _p(fx), len(fx), C.byref(prob), C.byref(ku), C.byref(mu)))

        def arr(ptr, n, t):
            return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(t)), shape=(n,)).copy() if n else np.zeros(0, np.dtype(t))
        K, P, E = prob.K, prob.P, prob.E
        a = dict(poses=arr(prob.poses, K * 7, C.c_double).reshape(K, 7), intr=arr(prob.intr, K * 4, C.c_double).reshape(K, 4),
                 fixed=arr(prob.fixed, K, C.c_uint8), points=arr(prob.points, P * 3, C.c_double).reshape(P, 3),
                 obs_kf=arr(prob.obs_kf, E, C.c_int32), obs_mp=arr(prob.obs_mp, E, C.c_int32), obs_uv=arr(prob.obs_uv, E * 2, C.c_float).reshape(E, 2),
                 obs_w=arr(prob.obs_w, E, C.c_float))
        return prob, a, arr(ku, K, C.c_uint64), arr(mu, P, C.c_uint64)
