"""RecForYouProcess.getRecList (online/recprocess/RecForYouProcess.java:29-105) restated literally in Python, on top of
oracle/similar_recall.py's catalogue.

* `DataManager.loadRatingData` (DataManager.java:208-242): userMap holds every userId of a 4-field ratings.csv line,
  whether or not the movie is known.  `getUserById` of anyone else is null, and getRecList returns an empty list.
* `loadUserEmb` (:144-164): a userEmb.csv line whose user is not in userMap is skipped; a later line of a user
  replaces the earlier one.
* The candidates are `getMovies(800, "rating")` (`RecallCatalogue.get_movies`: movieMap's HashMap order, stably
  sorted by averageRating descending).
* Rankers, the Java's `switch` strings (:72-88):
  - "emb": `calculateEmbSimilarScore`, `Embedding.calculateSimilarity` of the user's vector and the movie's: -1
    when the user has none, the movie has none or the dimensions differ; float products summed in double, so a zero
    vector gives NaN;
  - "nerualcf" (sic): the served model's score of each (userId, movieId) pair, from `score_fn(user_id, movie_ids)`;
    a pair outside the model's vocabulary makes TF-Serving reject the request, which `score_fn` reports by raising
    `ModelRange`, and the page is then empty (the Java throws);
  - anything else, the correctly spelled "neuralcf" included: `candidates.size() - i` for candidate i.
* The HashMap<Movie, Double> is sorted by `Double.compare` descending (NaN first) and cut to `size`.  Java leaves tied
  scores in identity-hash order; here they go by movie id ascending, as the similar-movies page does.
"""
from __future__ import annotations

import math

import numpy as np

from . import ctr_oracle as O
from . import similar_movies as S

OK, UNKNOWN_USER, MODEL_RANGE = 0, 1, 2
CANDIDATES = 800


class ModelRange(ValueError):
    """A (userId, movieId) pair outside the served model's vocabulary."""


def java_desc_key(x: float):
    """A sort key equal to the order of `Double.compare(b, a)`: NaN first, then +inf .. +0.0, then -0.0 .. -inf."""
    x = float(x)
    if x != x:
        return (0, 0.0, 0)
    return (1, -x, 1 if math.copysign(1.0, x) < 0 else 0)


def ctr_score_fn(spec, W, dtype=np.float32):
    """score_fn of the "nerualcf" ranker from oracle/ctr_oracle's NeuralCF / two-tower forward: the model output
    (the probability, or the raw dot of a two-tower model without its final Dense) of (user, movie) for each movie,
    as float64; ModelRange when the user or a movie is outside the spec's vocabulary."""
    if spec.model not in ("neuralcf", "twotowers"):
        raise ValueError("the nerualcf ranker needs a neuralcf or twotowers spec, not %r" % (spec.model,))

    def score(user_id, movie_ids):
        m = np.asarray(movie_ids, np.int64)
        if not 0 <= user_id < spec.n_users or (m.size and (m.min() < 0 or m.max() >= spec.n_movies)):
            raise ModelRange("user %d or a candidate outside the model" % user_id)
        feats = {"movieId": m.astype(np.int32), "userId": np.full(m.shape[0], user_id, np.int32)}
        return O.forward(spec, W, feats, dtype)[0].reshape(-1).astype(np.float64)
    return score


class RecForYou:
    """The page over `catalogue` (an oracle/similar_recall.RecallCatalogue), the ratings' userId column in file order
    and the userEmb.csv rows (ids, vectors) in file order (or None); a vector list may be any length.  `cosine(q, C)`
    scores the emb ranker: `similar_movies.java_cosine_many` (the Java's order) or `warp_cosine_many` (the device's)."""

    def __init__(self, catalogue, rating_user, user_emb_ids=None, user_emb=None, cosine=S.java_cosine_many):
        self.cat = catalogue
        self.cosine = cosine
        self.users = {int(u) for u in np.asarray(rating_user).tolist()}
        self.emb = {}
        if user_emb_ids is not None:
            for u, v in zip(np.asarray(user_emb_ids).tolist(), user_emb):
                if int(u) in self.users:
                    self.emb[int(u)] = np.asarray(v, np.float32)

    def candidates(self):
        """getMovies(800, "rating"), as slots."""
        return self.cat.get_movies(CANDIDATES, "rating")

    def scores(self, user_id, model, score_fn=None):
        """The ranker's score of each candidate, in candidate order."""
        cands = self.candidates()
        if model == "emb":
            uv = self.emb.get(int(user_id))
            have = [c for c in cands if uv is not None and c in self.cat.emb and len(self.cat.emb[c]) == len(uv)]
            s = dict(zip(have, self.cosine(uv, np.array([self.cat.emb[c] for c in have])) if have else []))
            return [float(s[c]) if c in s else -1.0 for c in cands]
        if model == "nerualcf":
            if score_fn is None:
                raise ValueError("the nerualcf ranker needs a score function")
            return [float(x) for x in score_fn(int(user_id), [self.cat.ids[c] for c in cands])]
        return [float(len(cands) - i) for i in range(len(cands))]

    def rec_list(self, user_id, size, model="emb", score_fn=None):
        """(ids, scores, status) of getRecList(user_id, size, model)."""
        if size < 1:
            raise ValueError("size must be >= 1, got %d" % size)
        if int(user_id) not in self.users:
            return [], [], UNKNOWN_USER
        try:
            scores = self.scores(user_id, model, score_fn)
        except ModelRange:
            return [], [], MODEL_RANGE
        items = sorted(zip(scores, (self.cat.ids[c] for c in self.candidates())),
                       key=lambda t: (java_desc_key(t[0]), t[1]))[:size]
        return [i for _, i in items], [s for s, _ in items], OK
