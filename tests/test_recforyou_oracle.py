"""oracle/recforyou.py, the literal restatement of RecForYouProcess.getRecList, against hand-worked cases: unknown users,
missing, zero and mismatched vectors, the default ranker and its spellings, short catalogues, the size cut, the
userEmb.csv rules and the tie and NaN order (DESIGN.md section 4.25)."""
import functools
import math

import numpy as np
import pytest

from oracle import recforyou as R
from oracle.ctr_oracle import java_double_compare
from oracle.similar_recall import RecallCatalogue


def _catalogue(n=5, emb=True):
    """Movies 10, 20, .. in load order; movie k's single rating is 5 - k / 2 (so rating order is load order), and
    every movie has a vector but the third."""
    ids = [10 * (k + 1) for k in range(n)]
    rm = ids
    rs = [5 - k / 2 for k in range(n)]
    vec = {10: [1, 0], 20: [0, 1], 40: [1, 1], 50: [-1, 0]}
    if not emb:
        return RecallCatalogue(ids, [["A"]] * n, rm, rs)
    eid = [i for i in ids if i in vec]
    return RecallCatalogue(ids, [["A"]] * n, rm, rs, eid, np.array([vec[i] for i in eid], np.float32))


def test_an_unknown_user_gets_an_empty_list():
    page = R.RecForYou(_catalogue(), [1, 1, 2], [1], [[1.0, 0.0]])
    for model in ("emb", "default", "nerualcf"):
        assert page.rec_list(3, 10, model, score_fn=lambda u, m: [0.5] * len(m)) == ([], [], R.UNKNOWN_USER)


def test_a_user_without_a_vector_scores_every_candidate_minus_one_in_id_order():
    cat = RecallCatalogue([30, 10, 20], [["A"]] * 3, [30, 10, 20], [1.0, 5.0, 3.0], [10, 20, 30],
                          np.eye(3, dtype=np.float32))
    page = R.RecForYou(cat, [7], None, None)
    ids, scores, st = page.rec_list(7, 10, "emb")
    assert st == R.OK and ids == [10, 20, 30] and scores == [-1.0] * 3


def test_a_zero_vector_puts_nan_first():
    page = R.RecForYou(_catalogue(), [1], [1], [[0.0, 0.0]])
    ids, scores, _ = page.rec_list(1, 10, "emb")
    # 0 / 0 for the four movies with vectors; -1 for movie 30, which has none
    assert ids == [10, 20, 40, 50, 30]
    assert all(math.isnan(s) for s in scores[:4]) and scores[4] == -1.0


def test_cosines_rank_descending():
    page = R.RecForYou(_catalogue(), [1], [1], [[1.0, 0.0]])
    ids, scores, _ = page.rec_list(1, 10, "emb")
    assert ids == [10, 40, 20, 30, 50]
    assert scores[0] == 1.0 and scores[1] == pytest.approx(1 / math.sqrt(2), abs=1e-15)
    assert scores[2:] == [0.0, -1.0, -1.0]          # 30 has no vector and 50 is opposite: a tie at -1, by id


def test_a_dimension_mismatch_scores_minus_one():
    page = R.RecForYou(_catalogue(), [1], [1], [[1.0, 0.0, 0.0]])
    ids, scores, _ = page.rec_list(1, 10, "emb")
    assert ids == [10, 20, 30, 40, 50] and scores == [-1.0] * 5


def test_a_movie_without_a_vector_scores_minus_one():
    page = R.RecForYou(_catalogue(emb=False), [1], [1], [[1.0, 2.0]])
    assert page.rec_list(1, 10, "emb")[1] == [-1.0] * 5
    page = R.RecForYou(_catalogue(), [1], [1], [[0.0, 1.0]])
    ids, scores, _ = page.rec_list(1, 10, "emb")
    assert dict(zip(ids, scores))[30] == -1.0


@pytest.mark.parametrize("model", ["default", "neuralcf", "", "EMB"])
def test_the_default_ranker_scores_size_minus_position(model):
    """Any string but "emb" and "nerualcf" - the correctly spelled "neuralcf" too - is the default branch."""
    cat = RecallCatalogue([30, 10, 20, 40], [["A"]] * 4, [30, 10, 20, 40], [4.0, 2.0, 5.0, 3.0])
    page = R.RecForYou(cat, [1], [1], [[1.0]])
    ids, scores, st = page.rec_list(1, 10, model)
    assert st == R.OK and ids == [20, 30, 40, 10] and scores == [4.0, 3.0, 2.0, 1.0]


def test_the_default_ranker_over_800_candidates_and_the_cut():
    n = 1000
    ids = list(range(1, n + 1))
    cat = RecallCatalogue(ids, [["A"]] * n, ids, [float(1 + (i * 7919) % 9) / 2 for i in ids])
    page = R.RecForYou(cat, [5])
    cands = page.candidates()
    assert len(cands) == 800
    out, scores, _ = page.rec_list(5, 2000, "default")
    assert out == [cat.ids[c] for c in cands] and scores == [800.0 - i for i in range(800)]
    assert page.rec_list(5, 1, "default") == ([cat.ids[cands[0]]], [800.0], R.OK)
    avg = [cat.avg[c] for c in cands]
    assert avg == sorted(avg, reverse=True) and min(avg) >= max(cat.avg[c] for c in set(range(n)) - set(cands))


def test_fewer_movies_than_800_and_size_past_the_candidates():
    page = R.RecForYou(_catalogue(), [1], [1], [[1.0, 0.0]])
    ids, scores, _ = page.rec_list(1, 9, "default")
    assert ids == [10, 20, 30, 40, 50] and scores == [5.0, 4.0, 3.0, 2.0, 1.0]
    assert page.rec_list(1, 1, "emb") == ([10], [1.0], R.OK)
    with pytest.raises(ValueError):
        page.rec_list(1, 0, "default")


def test_a_later_user_vector_line_wins_and_unknown_users_lines_are_ignored():
    page = R.RecForYou(_catalogue(), [1, 2], [1, 9, 1], [[1.0, 0.0], [0.0, 1.0], [0.0, 1.0]])
    assert set(page.emb) == {1}
    assert page.rec_list(1, 1, "emb")[0] == [20]
    assert page.rec_list(2, 10, "emb")[1] == [-1.0] * 5                # user 2 is known but has no vector
    assert page.rec_list(9, 10, "emb") == ([], [], R.UNKNOWN_USER)      # 9 has a vector but no rating


def test_nerualcf_takes_the_score_function_and_reports_model_range():
    page = R.RecForYou(_catalogue(), [1, 2], None, None)
    seen = []

    def score(u, movies):
        seen.append((u, list(movies)))
        if u == 2:
            raise R.ModelRange("user 2")
        return [0.25, 0.75, 0.25, float("nan"), 0.5]
    ids, scores, st = page.rec_list(1, 10, "nerualcf", score)
    assert seen == [(1, [10, 20, 30, 40, 50])]
    assert st == R.OK and ids == [40, 20, 50, 10, 30] and math.isnan(scores[0]) and scores[1:] == [0.75, 0.5, 0.25,
                                                                                                    0.25]
    assert page.rec_list(2, 10, "nerualcf", score) == ([], [], R.MODEL_RANGE)
    with pytest.raises(ValueError):
        page.rec_list(1, 10, "nerualcf")


def test_ctr_score_fn_range_rules():
    from sparrowrecsys_b200.spec import default_spec
    from sparrowrecsys_b200.weights import init_weights
    spec = default_spec("neuralcf", n_movies=60, n_users=5)
    fn = R.ctr_score_fn(spec, init_weights(spec, 1))
    s = fn(4, [10, 59])
    assert s.dtype == np.float64 and s.shape == (2,) and ((0 < s) & (s < 1)).all()
    for u, m in ((5, [10]), (-1, [10]), (0, [60]), (0, [-1, 3])):
        with pytest.raises(R.ModelRange):
            fn(u, m)
    with pytest.raises(ValueError):
        R.ctr_score_fn(default_spec("deepfm"), {})


def test_desc_key_is_double_compare_reversed():
    xs = [float("nan"), float("inf"), 1.0, 0.5, 0.0, -0.0, -1.0, float("-inf"), 0.5, -0.0, float("nan")]
    by_key = sorted(xs, key=R.java_desc_key)
    by_cmp = sorted(xs, key=functools.cmp_to_key(lambda a, b: java_double_compare(b, a)))
    assert [repr(x) for x in by_key] == [repr(x) for x in by_cmp]
