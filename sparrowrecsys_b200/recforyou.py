"""Recommended for you on the GPU: the reference's RecForYouService page, `RecForYouProcess.getRecList(userId, size,
model)` (online/recprocess/RecForYouProcess.java:29-105), for many users per call.

`RecForYou(catalogue, ratings, user_embeddings)` builds the user table once on the device
(`srs_recforyou_users_create_host`: DataManager.userMap's user ids and each user's userEmb.csv vector) over a
`similar.SimilarMovies` catalogue, whose getMovies(800, "rating") are the candidates; `recommend(user_ids, size,
model, ctr_model)` answers every user in one device call (`srs_recforyou_host`) with the "emb" ranker, the
"nerualcf" ranker (a NeuralCF or two-tower `CTRModel`) or the default one.  DESIGN.md section 4.25 gives the
semantics; oracle/recforyou.py restates the Java.  With the users' `uf:` hashes attached (`set_user_features`,
`srs_recforyou_users_set_features_host`) the "nerualcf" ranker takes every other CTR model too - DIN, DIEN, DeepFM,
DeepFM_v2, EmbeddingMLP, Wide&Deep - with its movie table (`CTRModel.set_movie_table`), through
`srs_recforyou_ctr_host` (DESIGN.md section 4.26).

    python -m sparrowrecsys_b200.recforyou movies.csv ratings.csv [--emb item2vecEmb.csv] [--user-emb userEmb.csv]
        [--model emb|nerualcf|default] [--savedmodel DIR [--savedmodel-kind neuralcf|twotowers]] --size N
        (--all | --user ID) [--data-manager-rows]
"""
from __future__ import annotations

import ctypes as C
from typing import List, Mapping, Optional, Sequence, Tuple

import numpy as np

from . import _lib
from .featureeng import load_movies_csv, load_ratings_csv
from .ranking import load_embeddings_csv
from .similar import SimilarList, SimilarMovies, _lists, data_manager_rows, data_manager_titles

OK, UNKNOWN_USER, MODEL_RANGE = _lib.SRS_RECFORYOU_OK, _lib.SRS_RECFORYOU_UNKNOWN_USER, _lib.SRS_RECFORYOU_MODEL_RANGE
STATUS_NAMES = {OK: "ok", UNKNOWN_USER: "unknown user", MODEL_RANGE: "outside the model"}


class RecForYou:
    """The "Recommended for you" page over a similar-movies catalogue, on the catalogue's device.

    `catalogue`: the `SimilarMovies` whose movies and ratings make DataManager's movieMap; it must stay open while this
    object is used.  `ratings`: the userId column of ratings.csv (as `featureeng.load_ratings_csv` returns it), which
    makes userMap.  `user_embeddings`: the (ids, vectors [n, dim]) of `ranking.load_embeddings_csv` on userEmb.csv, or
    None.  `device`: the catalogue's by default; the page needs both on one device."""

    def __init__(self, catalogue: SimilarMovies, ratings: Mapping[str, np.ndarray],
                 user_embeddings: Optional[Tuple[np.ndarray, np.ndarray]] = None, device: Optional[int] = None):
        users = np.ascontiguousarray(ratings["userId"], np.int32).reshape(-1)
        if user_embeddings is None:
            eid, emb, n_emb, dim = np.zeros(1, np.int32), np.zeros(1, np.float32), 0, 0
        else:
            eid = np.ascontiguousarray(user_embeddings[0], np.int32)
            emb = np.ascontiguousarray(user_embeddings[1], np.float32)
            if emb.ndim != 2 or emb.shape[0] != eid.shape[0] or (eid.shape[0] and emb.shape[1] < 1):
                raise ValueError("user embeddings: ids [n] and vectors [n, dim >= 1] expected, got %s and %s"
                                 % (eid.shape, emb.shape))
            n_emb, dim = eid.shape[0], (emb.shape[1] if eid.shape[0] else 0)
        self.catalogue = catalogue
        self.device = catalogue.device if device is None else int(device)
        self.dim = dim
        lib = _lib.load()
        h = C.c_void_p()
        p = lambda a: a.ctypes.data
        _lib.check(lib.srs_recforyou_users_create_host(p(users), users.shape[0], p(eid), p(emb), n_emb, dim,
                                                       self.device, C.byref(h)))
        self._h = h
        self.users = np.unique(users)
        self.has_user_features = False

    def set_user_features(self, store) -> None:
        """Attach the `uf:<userId>` hashes of `store` (a `featurestore.FeatureStore`) for every user of the table,
        typed by `parse_user_features` as `CTRModel.rank_user` types them; a user without a hash takes an empty
        hash's values.  Replaces what an earlier call attached."""
        from .features import genre_to_index
        from .featurestore import parse_user_features
        ids, genres, nums, hist = [], [], [], []
        for u in self.users.tolist():
            fields = store.user_features(u)
            if not fields:
                continue
            t = parse_user_features(fields)
            ids.append(u)
            genres.append([int(genre_to_index([t["userGenre%d" % (g + 1)]])[0]) for g in range(5)])
            nums.append([t["userAvgRating"], np.float32(t["userRatingCount"]), t["userRatingStddev"]])
            hist.append([t["userRatedMovie%d" % (k + 1)] for k in range(5)])
        n = len(ids)
        a = [np.ascontiguousarray(np.array(x, dt).reshape(shape)) for x, dt, shape in
             ((ids, np.int32, (n,)), (genres, np.int32, (n, 5)), (nums, np.float32, (n, 3)),
              (hist, np.int32, (n, 5)))]
        _lib.check(_lib.load().srs_recforyou_users_set_features_host(self._h, n, *[x.ctypes.data for x in a]))
        self.has_user_features = True

    def close(self) -> None:
        if getattr(self, "_h", None):
            _lib.load().srs_recforyou_users_destroy(self._h)
            self._h = None

    def __del__(self):
        self.close()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def recommend_arrays(self, user_ids, size: int, model: str = "emb", ctr_model=None):
        """One device call for every user: (ids int32 [U, size], scores float64 [U, size], count int32 [U], status
        int32 [U]); row u's first count[u] entries are its list, the rest 0.  `model` is the Java's string: "emb" the
        cosine ranker, "nerualcf" (sic) the served `ctr_model`, anything else - "neuralcf" included - the default
        ranker.  A NeuralCF or two-tower `ctr_model` reads (userId, movieId) only; any other kind reads the users'
        features (`set_user_features`) and its movie table (`CTRModel.set_movie_table`), and is ranked through
        `srs_recforyou_ctr_host`."""
        if self._h is None or self.catalogue._h is None:
            raise ValueError("the user table or its catalogue is closed")
        ctr = False
        if model == "emb":
            ranker, handle = _lib.SRS_RECFORYOU_EMB, None
        elif model == "nerualcf":
            if ctr_model is None:
                raise ValueError("the nerualcf ranker needs a CTRModel")
            if ctr_model.spec.model not in ("neuralcf", "twotowers"):
                if not self.has_user_features:
                    raise ValueError("a %s model reads the users' uf: features: call set_user_features first"
                                     % ctr_model.spec.model)
                if not getattr(ctr_model, "movie_table_rows", 0):
                    raise ValueError("a %s model reads movie features: call CTRModel.set_movie_table first"
                                     % ctr_model.spec.model)
                ctr = True
            ranker, handle = _lib.SRS_RECFORYOU_NEURALCF, ctr_model._h
        else:
            ranker, handle = _lib.SRS_RECFORYOU_DEFAULT, None
        q = np.ascontiguousarray(user_ids, np.int32).reshape(-1)
        size = int(size)
        if size < 1:
            raise ValueError("size must be >= 1, got %d" % size)
        U = q.shape[0]
        out = (np.zeros((U, size), np.int32), np.zeros((U, size), np.float64), np.zeros(U, np.int32),
               np.zeros(U, np.int32))
        p = lambda a: a.ctypes.data
        if ctr:
            _lib.check(_lib.load().srs_recforyou_ctr_host(self.catalogue._h, self._h, handle, p(q), U, size,
                                                          *map(p, out)))
        else:
            _lib.check(_lib.load().srs_recforyou_host(self.catalogue._h, self._h, handle, ranker, p(q), U, size,
                                                      *map(p, out)))
        return out

    def recommend(self, user_ids, size: int, model: str = "emb", ctr_model=None) -> List[SimilarList]:
        """getRecList(user_id, size, model) for each of `user_ids`; `status` is OK, UNKNOWN_USER or MODEL_RANGE."""
        return _lists(self.recommend_arrays(user_ids, size, model, ctr_model))


def main(argv: Sequence[str]) -> int:
    import argparse
    ap = argparse.ArgumentParser(prog="python -m sparrowrecsys_b200.recforyou")
    ap.add_argument("movies")
    ap.add_argument("ratings")
    ap.add_argument("--emb", help="item2vecEmb.csv: id:v v v ... lines")
    ap.add_argument("--user-emb", help="userEmb.csv: id:v v v ... lines")
    ap.add_argument("--model", default="emb", choices=("emb", "nerualcf", "default"),
                    help="the Java's ranker strings (nerualcf is its spelling)")
    ap.add_argument("--savedmodel", help="the served model for --model nerualcf: a shipped SavedModel directory")
    ap.add_argument("--savedmodel-kind", default="neuralcf", choices=("neuralcf", "twotowers"))
    ap.add_argument("--size", type=int, required=True)
    g = ap.add_mutually_exclusive_group(required=True)
    g.add_argument("--all", action="store_true", help="every user of ratings.csv, ascending")
    g.add_argument("--user", type=int)
    ap.add_argument("--data-manager-rows", action="store_true",
                    help="keep only the movies.csv lines the reference's DataManager loads (no comma in the title)")
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args(argv)
    if a.model == "nerualcf" and not a.savedmodel:
        ap.error("--model nerualcf needs --savedmodel")
    movies = load_movies_csv(a.movies)
    if a.data_manager_rows:
        keep = np.isin(movies["movieId"], data_manager_rows(a.movies))
        movies = {"movieId": movies["movieId"][keep], "genres": [x for x, k in zip(movies["genres"], keep) if k],
                  "title": data_manager_titles(a.movies)}
    ratings = load_ratings_csv(a.ratings)
    emb = load_embeddings_csv(a.emb) if a.emb else None
    uemb = load_embeddings_csv(a.user_emb) if a.user_emb else None
    users = np.unique(ratings["userId"]) if a.all else np.array([a.user], np.int32)
    ctr = None
    if a.model == "nerualcf":
        from .model import CTRModel
        ctr = CTRModel.from_savedmodel(a.savedmodel, a.savedmodel_kind, a.device)
    try:
        with SimilarMovies(movies, ratings, emb, a.device) as cat, RecForYou(cat, ratings, uemb) as page:
            for uid, r in zip(users.tolist(), page.recommend(users, a.size, a.model, ctr)):
                if r.status != OK:
                    print("%d\t(%s)" % (uid, STATUS_NAMES[r.status]))
                else:
                    print("%d\t%s" % (uid, " ".join("%d:%.17g" % (i, x) for i, x in zip(r.movie_ids.tolist(),
                                                                                        r.scores.tolist()))))
    finally:
        if ctr is not None:
            ctr.close()
    return 0


if __name__ == "__main__":
    import sys
    sys.exit(main(sys.argv[1:]))
