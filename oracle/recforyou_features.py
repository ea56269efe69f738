"""The "nerualcf" ranker of RecForYouProcess.getRecList (oracle/recforyou.py) with a served model that reads more than
(userId, movieId): DIN, DIEN, DeepFM, DeepFM_v2, EmbeddingMLP and Wide&Deep over the serving feature store
(DESIGN.md section 4.26).

Each (user, candidate) row is what `RecForYouProcess.java:46-52` posts with the user's `uf:<userId>` hash and the
movie's `mf:<movieId>` hash: `featurestore.assemble(user, store.user_features(user), candidates, movie_table,
hist_len=max(T, 5))`, scored by oracle/ctr_oracle's forward.  A user without a hash takes an empty hash's values.
`score_fn` raises `oracle.recforyou.ModelRange`, and the user's page is empty, exactly when predict would reject one
of the user's rows for range:
* the userId is outside the model;
* a stored history id the model reads is outside it: DIN and DIEN read userRatedMovie1..min(T, 5), Wide&Deep
  userRatedMovie1, the others none (the keys past 5 hold the padding id 0);
* a candidate is outside the model, or past the movie table.
DIN and DIEN pass movie ids through float32 before the check (DIN.py:95,125), so their rule does too.
"""
from __future__ import annotations

import numpy as np

from . import ctr_oracle as O
from .recforyou import ModelRange


def model_movie_id(spec, x: int) -> int:
    """A movie id as the forward range-checks it."""
    return int(np.float32(x)) if spec.model in ("din", "dien") else int(x)


def read_history_keys(spec):
    """The stored history keys (userRatedMovie1..5) that the model reads."""
    if spec.model in ("din", "dien"):
        return ["userRatedMovie%d" % k for k in range(1, min(spec.hist_len, 5) + 1)]
    return ["userRatedMovie1"] if spec.model == "widendeep" else []


def history_positions(spec):
    """The position of userRatedMovie1..5 among the model's history inputs, -1 where it does not read the key: DIN
    and DIEN read `spec.history_keys(T)`, the keys userRatedMovie1..T in ASCII order (so from T = 10 on
    userRatedMovie2 follows userRatedMovie1x); Wide&Deep reads userRatedMovie1; the others none."""
    from sparrowrecsys_b200.spec import history_keys
    if spec.model == "widendeep":
        return [0, -1, -1, -1, -1]
    if spec.model not in ("din", "dien"):
        return [-1] * 5
    keys = history_keys(spec.hist_len)
    return [keys.index("userRatedMovie%d" % k) if k <= spec.hist_len else -1 for k in range(1, 6)]


def feature_score_fn(spec, W, store, movie_table, dtype=np.float32):
    """score_fn of the "nerualcf" ranker (oracle/recforyou.RecForYou.rec_list) for a model over the `uf:` / `mf:`
    features of `store` (a featurestore.FeatureStore) and `movie_table` (a featurestore.MovieFeatureTable): the
    model output of each (user, movie) row as float64, or ModelRange under the rule above."""
    from sparrowrecsys_b200 import featurestore as FS
    if spec.model in ("neuralcf", "twotowers"):
        raise ValueError("a %s model reads (userId, movieId) only: use recforyou.ctr_score_fn" % spec.model)
    T = max(spec.hist_len, 5)

    def score(user_id, movie_ids):
        m = np.asarray(movie_ids, np.int64).reshape(-1)
        if not 0 <= user_id < spec.n_users:
            raise ModelRange("user %d outside the model" % user_id)
        for x in m.tolist():
            if not 0 <= model_movie_id(spec, x) < spec.n_movies or not 0 <= x < movie_table.n_movies:
                raise ModelRange("candidate %d outside the model or past the movie table" % x)
        fields = store.user_features(user_id)
        typed = FS.parse_user_features(fields, T)
        for k in read_history_keys(spec):
            if not 0 <= model_movie_id(spec, typed[k]) < spec.n_movies:
                raise ModelRange("user %d: %s = %d outside the model" % (user_id, k, typed[k]))
        feats = FS.assemble(user_id, fields, m.astype(np.int32), movie_table, hist_len=T)
        return O.forward(spec, W, feats, dtype)[0].reshape(-1).astype(np.float64)
    return score
