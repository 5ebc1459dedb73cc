"""Writes tests/golden/kfdb_queries.npz: every query of every scene of tests/kfdb_scenes.py under the six scoring types, as the
oracle answers it (returned uids, scored list with shared words and f64 scores):  python -m tests.golden.make_kfdb_golden

Before writing, the generator asserts that the oracle agrees with the independent numpy restatements of the scores and of the three
queries' counting / scoring steps (and the selection), and, where it is built, with the reference's own Database.cpp."""
import os

import numpy as np

from oracle import pykfdb
from tests import kfdb_scenes
from tests import test_kfdb_cpu as T

if __name__ == "__main__":
    for scoring in kfdb_scenes.SCORINGS:
        T.test_oracle_scores_equal_a_numpy_restatement(scoring)
    for name in sorted(T.SCENES):
        T.test_oracle_queries_equal_a_restatement_and_select(name)
        if pykfdb.Reference.available():
            for scoring in kfdb_scenes.SCORINGS:
                T.test_oracle_equals_the_reference_database(name, scoring)
    np.savez_compressed(T.GOLDEN, **T.golden_results())
    print(T.GOLDEN, os.path.getsize(T.GOLDEN))
