"""Regenerate the DIEN evaluate test set from a checkout of the reference SparrowRecSys repository.

    python tests/golden/make_dien_golden.py <reference checkout>

Writes `dien_testset.npz` next to this file: every column of the reference's
`src/main/resources/webroot/sampledata/testSamples.csv` that DIEN.py's model reads (DIEN.py:57-88), for all
22 440 rows in file order, as `features.load_samples_csv` types them, with `userGenre1` / `movieGenre1` as
vocabulary indices (-1 = missing).  The negative samples are not stored: `features.negative_history(...,
seed=2021)` draws them from `userRatedMovie2..5` the way DIEN.py:30-50 does.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from sparrowrecsys_b200 import features                              # noqa: E402
from sparrowrecsys_b200.spec import NUMERIC_KEYS, history_keys        # noqa: E402


def main(ref):
    full = features.load_samples_csv(os.path.join(ref, "src/main/resources/webroot/sampledata/testSamples.csv"))
    out = {k: full[k] for k in ("movieId", "userId", "label", *history_keys(5), *NUMERIC_KEYS)}
    for k in ("userGenre1", "movieGenre1"):
        out[k] = features.genre_to_index(full[k]).astype(np.int8)
    assert out["movieId"].shape[0] == 22440
    np.savez_compressed(os.path.join(HERE, "dien_testset.npz"), **out)


if __name__ == "__main__":
    main(sys.argv[1])
