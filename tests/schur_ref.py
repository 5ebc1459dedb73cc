"""A plain f64 restatement of the reduced camera system, numpy only (test infrastructure).

From the linear system of one state -- Hpp, bp, Hll, bl and W, in the layout of ccm_ba_debug_build / orc_ba_build -- it forms

    S        = blockdiag(Hpp + lam I) - sum_l W_l (Hll_l + lam I)^-1 W_l^T      over the free poses,
    b_schur  = bp - sum_l W_l (Hll_l + lam I)^-1 bl_l,
    dx_l     = (Hll_l + lam I)^-1 (bl_l - sum_a W_la^T x_a)                      for a given pose step x,

with the signs and the placement of lambda of the oracle's BlockSolver restatement (oracle/ba_oracle.cpp solve_system).  The landmark
inverse goes through the reference's own Cholesky D_l = U_l^T U_l: Z_e = W_e U_l^-1, g_l = U_l^-T bl_l, so that S = diag - sum Z Z^T.

Every entry gets its own tolerance TAU * bound.  The bound of an S entry is delta_ab (|Hpp| + lam) + A_ab with
A_ab = sum_l kappa_l |Z_al| |Z_bl|^T: a correct f64 kernel may sum the products in any order and may take its own (equally correct)
Cholesky factor, and kappa_l = || |U_l| |U_l^-1| ||_inf >= 1 is the factor by which a different rounding of U_l can move Z.  The same
construction with |g_l| bounds b_schur, and with |U_l^-1| (|g_l| + sum |Z_e|^T |x_a|) bounds dx_l.  A wrong, missing, transposed or
misplaced product exceeds its bound by many orders of magnitude (tests/test_schur_ref.py shows it).

Products are formed chunk by chunk over landmarks of equal observation count, so cfg5 at 1/10 length (2e7 products) fits in memory.
"""
from __future__ import annotations

import numpy as np

TAU = 1e-12
_CHUNK = 1 << 18   # products per batch


def _free_slots(p):
    return np.asarray(p.fixed) == 0


def _edge_mask(p):
    """(in_pattern, active): observations of free poses form the pattern of S (also inactive ones, like the device's bitmap);
    only active ones (edge flag bit 0 clear) contribute products"""
    free = _free_slots(p)
    kf = np.asarray(p.obs_kf)
    on_free = free[kf]
    flags = np.zeros(p.E, np.uint8) if p.edge_flags is None else np.asarray(p.edge_flags)
    active = (flags & 1) == 0
    return on_free, active


class SchurRef:
    """S, b_schur and their bounds, once per (state, lambda); dx_point on demand for a pose step."""

    def __init__(self, p, build, lam):
        K, P = p.K, p.P
        self.K, self.P, self.lam = K, P, float(lam)
        Hll = np.asarray(build["Hll"], np.float64)
        D = Hll + lam * np.eye(3)[None]
        U = np.swapaxes(np.linalg.cholesky(D), -1, -2)            # D = U^T U, U upper
        Uinv = np.linalg.inv(U)
        self.Uinv = Uinv
        self.kappa = np.maximum(1.0, (np.abs(U) @ np.abs(Uinv)).sum(-1).max(-1))
        self.g = np.einsum("lkj,lk->lj", Uinv, np.asarray(build["bl"], np.float64))   # U^-T bl
        on_free, active = _edge_mask(p)
        kf = np.asarray(p.obs_kf, np.int64)
        mp = np.asarray(p.obs_mp, np.int64)
        W = np.asarray(build["W"], np.float64)
        Z = W @ Uinv[mp]                                          # (E,6,3)
        Z[~active] = 0.0
        self.Z = Z
        sel = np.flatnonzero(on_free)
        sel = sel[np.lexsort((kf[sel], mp[sel]))]                 # by landmark, then pose
        self.sel, self.sel_active = sel, active[sel]
        e_kf, e_mp = kf[sel], mp[sel]
        assert not np.any((e_mp[1:] == e_mp[:-1]) & (e_kf[1:] == e_kf[:-1])), "a pose observes a landmark twice"
        free = _free_slots(p)
        Hpp = np.asarray(build["Hpp"], np.float64)
        # ---- upper blocks: pattern, sum of products, bound
        cnt = np.bincount(e_mp, minlength=P)
        start = np.concatenate([[0], np.cumsum(cnt)])
        groups = []
        keys_all = [np.flatnonzero(free) * (K + 1)]               # every free pose has its diagonal block
        for n in np.unique(cnt[cnt > 0]):
            ls = np.flatnonzero(cnt == n)
            iu, ju = np.triu_indices(n)
            idx = start[ls][:, None] + np.arange(n)[None, :]       # (L, n) positions in sel
            groups.append((ls, idx, iu, ju))
            keys_all.append(np.unique(e_kf[idx[:, iu]] * K + e_kf[idx[:, ju]]))
        keys = np.unique(np.concatenate(keys_all))
        nb = keys.size
        acc = np.zeros(nb * 36); bnd = np.zeros(nb * 36)
        Zs, Zabs = Z[sel], np.abs(Z[sel])
        ksel = self.kappa[e_mp]
        for ls, idx, iu, ju in groups:
            per = max(1, _CHUNK // len(iu))
            for c0 in range(0, len(ls), per):
                ii, jj = idx[c0:c0 + per][:, iu].ravel(), idx[c0:c0 + per][:, ju].ravel()
                bid = np.searchsorted(keys, e_kf[ii] * K + e_kf[jj])
                flat = (bid[:, None] * 36 + np.arange(36)[None, :]).ravel()
                prod = Zs[ii] @ np.swapaxes(Zs[jj], -1, -2)
                pabs = (Zabs[ii] @ np.swapaxes(Zabs[jj], -1, -2)) * ksel[ii][:, None, None]
                acc += np.bincount(flat, weights=prod.ravel(), minlength=nb * 36)
                bnd += np.bincount(flat, weights=pabs.ravel(), minlength=nb * 36)
        acc = acc.reshape(nb, 6, 6); bnd = bnd.reshape(nb, 6, 6)
        ua, ub = keys // K, keys % K
        diag = ua == ub
        up = -acc
        up[diag] += Hpp[ua[diag]] + lam * np.eye(6)[None]
        bnd[diag] += np.abs(Hpp[ua[diag]]) + lam * np.eye(6)[None]
        # ---- full symmetric pattern as block CSR in pose indices (the layout of ccm_ba_debug_schur_blocks)
        off = ~diag
        rows = np.concatenate([ua, ub[off]]); cols = np.concatenate([ub, ua[off]])
        vals = np.concatenate([up, np.swapaxes(up[off], -1, -2)])
        tols = np.concatenate([bnd, np.swapaxes(bnd[off], -1, -2)]) * TAU
        o = np.lexsort((cols, rows))
        self.col, self.val, self.tol = cols[o].astype(np.int32), vals[o], tols[o]
        self.row = rows[o]
        self.rowptr = np.searchsorted(self.row, np.arange(K + 1)).astype(np.int32)
        # ---- b_schur
        zg = np.einsum("erk,ek->er", Zs, self.g[e_mp])
        zgabs = np.einsum("erk,ek->er", Zabs, np.abs(self.g[e_mp])) * ksel[:, None]
        bp = np.asarray(build["bp"], np.float64)
        coeff = np.stack([np.bincount(e_kf, weights=zg[:, r], minlength=K) for r in range(6)], 1)
        cb = np.stack([np.bincount(e_kf, weights=zgabs[:, r], minlength=K) for r in range(6)], 1)
        self.bschur = np.where(free[:, None], bp - coeff, 0.0)
        self.bschur_tol = np.where(free[:, None], np.abs(bp) + cb, 0.0) * TAU

    # ---- views ------------------------------------------------------------------------------------------------------
    def dense(self):
        n = 6 * self.K
        S = np.zeros((n, n)); T = np.zeros((n, n))
        for q in range(self.col.size):
            a, b = self.row[q], self.col[q]
            S[6 * a:6 * a + 6, 6 * b:6 * b + 6] = self.val[q]
            T[6 * a:6 * a + 6, 6 * b:6 * b + 6] = self.tol[q]
        return S, T


def _bind_dx(ref, p):
    kf = np.asarray(p.obs_kf, np.int64); mp = np.asarray(p.obs_mp, np.int64)
    e = ref.sel[ref.sel_active]
    Ze, ke, le = ref.Z[e], kf[e], mp[e]

    def dx(x):
        x = np.asarray(x, np.float64).reshape(ref.K, 6)
        zx = np.einsum("erk,er->ek", Ze, x[ke])
        zxa = np.einsum("erk,er->ek", np.abs(Ze), np.abs(x[ke]))
        s = np.stack([np.bincount(le, weights=zx[:, k], minlength=ref.P) for k in range(3)], 1)
        sa = np.stack([np.bincount(le, weights=zxa[:, k], minlength=ref.P) for k in range(3)], 1)
        d = np.einsum("ljk,lk->lj", ref.Uinv, ref.g - s)
        t = np.einsum("ljk,lk->lj", np.abs(ref.Uinv), np.abs(ref.g) + sa) * ref.kappa[:, None] * TAU
        return d, t
    return dx


def schur_reference(p, build, lam):
    """SchurRef of the state `build` describes (ccm_ba_debug_build / orc_ba_build output of problem p) at damping lam"""
    ref = SchurRef(p, build, lam)
    ref.dx_point = _bind_dx(ref, p)   # dx_point(x) -> (dx (P,3), tolerance (P,3)) for the pose step x (K,6)
    return ref


def ratio(err, tol):
    """max of |err| / tol over the entries; an entry with zero tolerance must be exactly zero"""
    err = np.abs(np.asarray(err, np.float64)); tol = np.asarray(tol, np.float64)
    bad_zero = (tol == 0) & (err != 0)
    if bad_zero.any():
        return float("inf")
    r = np.divide(err, tol, out=np.zeros_like(err), where=tol > 0)
    return float(r.max()) if r.size else 0.0


def compare_blocks(ref, got):
    """err / tol of a block-CSR export (ccm_ba_debug_schur_blocks) against the reference; the patterns must be identical"""
    assert np.array_equal(got["rowptr"], ref.rowptr), "row pattern of S differs"
    assert np.array_equal(got["col"], ref.col), "column pattern of S differs"
    return dict(S=ratio(got["val"] - ref.val, ref.tol), bschur=ratio(got["bschur"] - ref.bschur, ref.bschur_tol))


def worst_block(ref, got):
    """(row, col, err/tol) of the worst block: what a failing comparison names"""
    err = np.abs(got["val"] - ref.val)
    r = np.where(ref.tol > 0, err / np.where(ref.tol > 0, ref.tol, 1.0), np.where(err > 0, np.inf, 0.0)).reshape(len(err), -1).max(1)
    q = int(np.argmax(r))
    return int(ref.row[q]), int(ref.col[q]), float(r[q])
