"""Bytes k_pcg2 streams per iteration, from a problem's S pattern, against the full block-CSR (nnzb * 288).

Restates in numpy what pcg2_plan (csrc/pcg2.cuh) builds at create time:
  * the CTA cut: one CTA per SM (at most ceil(items / 16)), contiguous rows balanced by the items of the FULL rows;
  * the skip rule: inside a CTA's rows [c0, c1), an upper block (a, b) with a < b < c1 is applied transposed by the lane pair that
    streams it, and its mirror (b, a) is not streamed;
  * the slab spans: a warp adds S_ab^T p_a into a slab of SLAB_ROWS rows from the lowest row b it serves; a block beyond that is not
    applied transposed and its mirror is streamed again, which moves the warps' runs, so the plan is redone until nothing moves.

Usage: python tools/pcg2_bytes.py cfg5 loop_closure ...   (a name of synth.CONFIGS or of tests/schur_setup_scenes.SCENES)
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ITEM_BLOCKS, REC, WARPS, SLAB_ROWS = 16, 20, 16, 48
NO_SLAB = -(1 << 30)


def pattern(p):
    """full block-CSR pattern of S in slot order: rowptr (Kf + 1,), col (nnzb,)"""
    sys.path.insert(0, ROOT)
    from tests import schur_setup_scenes as SC
    a, b = SC.covis_pairs(p)
    Kf = SC.free_poses(p).size
    r = np.concatenate([a, b[a != b]]); c = np.concatenate([b, a[a != b]])
    o = np.lexsort((c, r))
    r, c = r[o], c[o]
    return np.searchsorted(r, np.arange(Kf + 1)), c.astype(np.int64)


def cta_cut(rowptr, sms=132):
    full = -(-np.diff(rowptr) // ITEM_BLOCKS)
    row_item = np.concatenate([[0], np.cumsum(full)])
    n = int(row_item[-1])
    grid = max(1, min(sms, -(-n // WARPS)))
    want = np.array([n * c // grid for c in range(grid)], np.int64)
    cut = np.minimum(np.searchsorted(row_item, want, side="left"), len(full))
    cut[0] = 0
    return np.concatenate([cut, [len(full)]])


def plan(rowptr, col, cta_row):
    """items (n, 20), cta_item (grid + 1,), slab_lo (grid, 16), streamed blocks"""
    Kf, nnzb, grid = len(rowptr) - 1, len(col), len(cta_row) - 1
    row = np.repeat(np.arange(Kf), np.diff(rowptr))
    cta = np.searchsorted(cta_row, row, side="right") - 1
    cand = (col > row) & (col < cta_row[cta + 1])
    keys = row * Kf + col
    mirror = np.full(nnzb, -1, np.int64)
    mirror[cand] = np.searchsorted(keys, col[cand] * Kf + row[cand])
    mirrored = cand.copy()
    j = np.arange(nnzb)
    row_start = np.zeros(nnzb, bool); row_start[rowptr[:-1][np.diff(rowptr) > 0]] = True
    while True:
        skip = np.zeros(nnzb, bool); skip[mirror[mirrored]] = True
        run_first = row_start | np.concatenate([[True], skip[:-1]])
        run0 = np.maximum.accumulate(np.where(run_first, j, 0))
        start = ~skip & ((j - run0) % ITEM_BLOCKS == 0)
        item = np.cumsum(start) - 1
        s_j = j[start]
        n = s_j.size
        nb = np.bincount(item[~skip], minlength=n)
        irow = row[s_j]
        cta_item = np.searchsorted(irow, cta_row)
        # warp of every item: the kernel's runs it0 + (it1 - it0) * w / 16
        warp = np.zeros(n, np.int64)
        for c in range(grid):
            it0, it1 = cta_item[c], cta_item[c + 1]
            for w in range(WARPS):
                warp[it0 + (it1 - it0) * w // WARPS: it0 + (it1 - it0) * (w + 1) // WARPS] = c * WARPS + w
        tr = mirrored & ~skip
        slab = np.full(grid * WARPS, np.iinfo(np.int64).max)
        np.minimum.at(slab, warp[item[tr]], col[tr])
        out = tr & (col - slab[warp[np.maximum(item, 0)]] >= SLAB_ROWS)
        if not out.any():
            break
        mirrored &= ~out
    items = np.zeros((n, REC), np.int64)
    items[:, 0], items[:, 1], items[:, 2] = s_j, nb, irow
    k = j - s_j[np.maximum(item, 0)]
    sj = ~skip
    items[item[sj], 4 + k[sj]] = col[sj]
    np.bitwise_or.at(items[:, 3], item[tr], 1 << (4 + k[tr]))
    first = np.concatenate([[True], irow[1:] != irow[:-1]]) if n else np.zeros(0, bool)
    last = np.concatenate([irow[1:] != irow[:-1], [True]]) if n else np.zeros(0, bool)
    items[:, 3] |= first * 1 | last * 2
    slab_lo = np.where(slab == np.iinfo(np.int64).max, NO_SLAB, slab).reshape(grid, WARPS)
    return dict(items=items, cta_item=cta_item, slab_lo=slab_lo, streamed=int(sj.sum()))


def report(name, p, sms=132):
    rowptr, col = pattern(p)
    cta_row = cta_cut(rowptr, sms)
    P = plan(rowptr, col, cta_row)
    nnzb, n = len(col), len(P["items"])
    return dict(problem=name, Kf=len(rowptr) - 1, nnzb=nnzb, ctas=len(cta_row) - 1, items=n, streamed_blocks=P["streamed"],
                streamed_bytes=P["streamed"] * 288 + n * REC * 4, full_bytes=nnzb * 288,
                ratio=round((P["streamed"] * 288 + n * REC * 4) / (nnzb * 288), 4),
                transposed_blocks=int(sum(bin(int(f) >> 4).count("1") for f in P["items"][:, 3])))


def problem(name):
    sys.path.insert(0, ROOT)
    from ccm_slam_b200 import synth
    if name in synth.CONFIGS:
        return synth.make_config(name)
    from tests import schur_setup_scenes as SC
    return SC.SCENES[name]()


if __name__ == "__main__":
    for name in sys.argv[1:] or ["cfg5"]:
        print(json.dumps(report(name, problem(name))), flush=True)
