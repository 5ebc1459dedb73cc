"""The numpy restatement of k_pcg2's item plan (tools/pcg2_bytes.py) on the CPU: with four CTAs on cfg5 at 1/10 length some warps
serve rows beyond their slab, so those blocks fall back to the full stream while the plan still mirrors the others.  The device's plan
is compared with this restatement block for block in tests/test_gpu_pcg2_mirror.py."""
import os
import sys

import numpy as np

from ccm_slam_b200 import synth

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import pcg2_bytes as PB  # noqa: E402


def test_the_four_cta_case_falls_back():
    p = synth.make_config("cfg5", K=1000, P=100000)
    rowptr, col = PB.pattern(p)
    cut = PB.cta_cut(rowptr, sms=4)
    row = np.repeat(np.arange(len(rowptr) - 1), np.diff(rowptr))
    cta = np.searchsorted(cut, row, side="right") - 1
    cand = int(((col > row) & (col < cut[cta + 1])).sum())
    P = PB.plan(rowptr, col, cut)
    tr = int(sum(bin(int(f) >> 4).count("1") for f in P["items"][:, 3]))
    assert 0 < tr < cand
    # every block is streamed once or applied as the transpose of a streamed block
    assert P["streamed"] + tr == len(col)
