"""ctypes binding of include/srs_ctr.h (the whole FFI surface, nothing else).

The library is built in-tree by `sparrowrecsys_b200.build`; loading fails loudly if
it is missing - there is no CPU or PyTorch fallback for the forward path.
"""
from __future__ import annotations

import ctypes as C
import os

from . import build as _build

SRS_OK = 0
SRS_ERR_INVALID, SRS_ERR_MISSING, SRS_ERR_SHAPE = -1, -2, -3
SRS_ERR_CUDA, SRS_ERR_RANGE, SRS_ERR_NOMEM = -4, -5, -6
SRS_HOST, SRS_DEVICE_BORROWED = 0, 1
ABI_VERSION = 4


class SrsSpec(C.Structure):
    _fields_ = [("kind", C.c_int32), ("emb_dim", C.c_int32), ("n_movies", C.c_int32),
                ("n_users", C.c_int32), ("n_genres", C.c_int32), ("hist_len", C.c_int32),
                ("n_hidden", C.c_int32), ("hidden", C.c_int32 * 4), ("au_hidden", C.c_int32),
                ("cross_buckets", C.c_int32), ("proj_dim", C.c_int32), ("final_dense", C.c_int32)]


class SrsTensor(C.Structure):
    _fields_ = [("name", C.c_char_p), ("data", C.c_void_p), ("rows", C.c_int64),
                ("cols", C.c_int64), ("location", C.c_int32)]


class SrsBatch(C.Structure):
    _fields_ = [("B", C.c_int32), ("hist_stride", C.c_int32), ("movie_id", C.c_void_p),
                ("user_id", C.c_void_p), ("hist", C.c_void_p), ("movie_genre", C.c_void_p),
                ("user_genre", C.c_void_p), ("numerics", C.c_void_p), ("hist16", C.c_void_p)]


EXPORTS = ("srs_abi_version", "srs_last_error", "srs_model_create", "srs_model_create_ex", "srs_model_destroy",
           "srs_predict_device", "srs_predict_host", "srs_predict_host_batches", "srs_num_slots", "srs_predict_host_async",
           "srs_wait_slot", "srs_model_status", "srs_model_bytes_per_inference",
           "srs_model_kernel_name", "srs_model_set_sm_limit", "srs_launch_count", "srs_fill_uniform",
           "srs_cosine_scores_device", "srs_topk_device", "srs_rank_host", "srs_gather_create", "srs_gather_export",
           "srs_gather_connect", "srs_gather_destroy", "srs_predict_device_gather", "srs_gather_wait",
           "srs_gather_scores", "srs_gather_copy_scores", "srs_model_set_movie_features", "srs_rank_user_host",
           "srs_selftest_wgmma", "srs_metrics_create", "srs_metrics_destroy", "srs_metrics_reset",
           "srs_metrics_update_device", "srs_metrics_result", "srs_evaluate_host_batches",
           "srs_dien_outputs_device", "srs_dien_outputs_host_batches", "srs_dien_evaluate_host_batches",
           "srs_trainer_create", "srs_trainer_create_ex", "srs_trainer_create_any", "srs_trainer_destroy", "srs_trainer_fit_host", "srs_trainer_get_weights",
           "srs_trainer_iterations", "srs_trainer_fit_validate_host", "srs_trainer_evaluate_host", "srs_trainer_fit_dien_host",
           "srs_trainer_fit_weighted_host", "srs_trainer_evaluate_weighted_host", "srs_evaluate_weighted_host_batches",
           "srs_metrics_update_weighted_device",
           "srs_featureeng_host", "srs_item2vec_host", "srs_user_embeddings_host", "srs_als_fit_host",
           "srs_als_fit_folds_host", "srs_als_recommend_host", "srs_item_transitions_host", "srs_random_walks_host",
           "srs_graph_embedding_host", "srs_lsh_transform_host", "srs_lsh_query_host", "srs_approx_quantile_host",
           "srs_quantile_discretizer_host", "srs_bucketize_host", "srs_minmax_scale_host", "srs_rating_features_host",
           "srs_string_indexer_host", "srs_genre_multihot_host", "srs_sample_split_host",
           "srs_sample_split_by_timestamp_host", "srs_als_fit_implicit_host", "srs_ranking_metrics_host",
           "srs_als_fit_nonnegative_host", "srs_als_fit_folds_nonnegative_host", "srs_lsh_similarity_join_host",
           "srs_binary_metrics_create_host", "srs_binary_metrics_create_device", "srs_binary_metrics_destroy",
           "srs_binary_metrics_summary", "srs_binary_metrics_curve", "srs_binary_metrics_confusion",
           "srs_similar_catalog_create_host", "srs_similar_movies_host", "srs_similar_catalog_destroy",
           "srs_similar_catalog_create_ex_host", "srs_similar_movies_candidates_host",
           "srs_similar_embedding_recall_host", "srs_recforyou_users_create_host", "srs_recforyou_users_destroy",
           "srs_recforyou_host", "srs_recforyou_users_set_features_host", "srs_recforyou_ctr_host")

_lib = None


class SrsUserRow(C.Structure):
    """`srs_user_row` (include/srs_ctr.h): the typed `uf:<userId>` hash of one user."""
    _fields_ = [("user_id", C.c_int32), ("user_genre", C.c_int32 * 5), ("user_numerics", C.c_float * 3),
                ("n_hist", C.c_int32), ("hist", C.c_void_p)]


class SrsEvalResult(C.Structure):
    """`srs_eval_result` (include/srs_ctr.h): what `model.evaluate` reports, with its counts."""
    _fields_ = [("rows", C.c_int64), ("positives", C.c_int64), ("correct", C.c_int64), ("loss", C.c_double),
                ("accuracy", C.c_double), ("roc_auc", C.c_double), ("pr_auc", C.c_double)]


class SrsDienEvalResult(C.Structure):
    """`srs_dien_eval_result` (include/srs_ctr.h): what DIEN's `model.evaluate` reports (DIEN.py:304)."""
    _fields_ = [("rows", C.c_int64), ("batches", C.c_int64), ("loss", C.c_double), ("auc", C.c_double),
                ("auc_value", C.c_double)]


class SrsAdam(C.Structure):
    """`srs_adam` (include/srs_ctr.h): Keras Adam's hyper-parameters."""
    _fields_ = [("lr", C.c_float), ("beta_1", C.c_float), ("beta_2", C.c_float), ("epsilon", C.c_float)]


class SrsSamples(C.Structure):
    """`srs_samples` (include/srs_ctr.h): the output columns of srs_featureeng_host."""
    _fields_ = [(name, C.c_void_p) for name in (
        "row", "label", "release_year", "movie_genre", "movie_rating_count", "movie_avg_rating",
        "movie_rating_stddev", "user_rated_movie", "user_rating_count", "user_avg_release_year",
        "user_release_year_stddev", "user_avg_rating", "user_rating_stddev", "user_genre")]


class SrsItem2vecParams(C.Structure):
    """`srs_item2vec_params` (include/srs_ctr.h): Word2Vec's settings."""
    _fields_ = [("vector_size", C.c_int32), ("window", C.c_int32), ("iterations", C.c_int32),
                ("partitions", C.c_int32), ("seed", C.c_uint64)]


class SrsAlsParams(C.Structure):
    """`srs_als_params` (include/srs_ctr.h): ALS's settings."""
    _fields_ = [("rank", C.c_int32), ("max_iter", C.c_int32), ("reg_param", C.c_double), ("seed", C.c_uint64)]


class SrsAlsModel(C.Structure):
    """`srs_als_model` (include/srs_ctr.h): one model of a batched ALS fit."""
    _fields_ = [("rank", C.c_int32), ("max_iter", C.c_int32), ("reg_param", C.c_double),
                ("exclude_fold", C.c_int32)]


class SrsBinarySummary(C.Structure):
    """`srs_binary_summary` (include/srs_ctr.h): one score set of BinaryClassificationMetrics."""
    _fields_ = [("n", C.c_int64), ("positives", C.c_int64), ("negatives", C.c_int64), ("thresholds", C.c_int64),
                ("area_under_roc", C.c_double), ("area_under_pr", C.c_double)]


SRS_BM_ROC, SRS_BM_PR, SRS_BM_THRESHOLDS, SRS_BM_PRECISION, SRS_BM_RECALL, SRS_BM_FMEASURE = range(6)
SRS_SIMILAR_DEFAULT, SRS_SIMILAR_EMB = 0, 1
SRS_SIMILAR_OK, SRS_SIMILAR_UNKNOWN_MOVIE, SRS_SIMILAR_NO_EMBEDDING = 0, 1, 2
SRS_SIMILAR_CANDIDATES_GENRE, SRS_SIMILAR_CANDIDATES_MULTIPLE = 0, 1
SRS_RECFORYOU_DEFAULT, SRS_RECFORYOU_EMB, SRS_RECFORYOU_NEURALCF = 0, 1, 2
SRS_RECFORYOU_OK, SRS_RECFORYOU_UNKNOWN_USER, SRS_RECFORYOU_MODEL_RANGE = 0, 1, 2


class SrsError(RuntimeError):
    def __init__(self, code, message):
        super().__init__("srs error %d: %s" % (code, message))
        self.code = code


class SrsInvalidError(SrsError, ValueError):
    """SRS_ERR_INVALID: an argument the library does not support (e.g. a hidden width past a builder's limit)."""


def lib_path() -> str:
    # SRS_CTR_LIB: an alternative build of the library (kernel-tuning experiments)
    return os.environ.get("SRS_CTR_LIB") or _build.LIB


def load():
    """dlopen libsrs_ctr.so (no CUDA call is made here) and declare signatures."""
    global _lib
    if _lib is not None:
        return _lib
    path = lib_path()
    if not os.path.exists(path):
        raise ImportError(
            "%s not found: build it with `python -m sparrowrecsys_b200.build` "
            "(needs nvcc; there is no CPU fallback for the CTR forward path)" % path)
    lib = C.CDLL(path)
    lib.srs_abi_version.restype = C.c_int
    lib.srs_last_error.restype = C.c_char_p
    lib.srs_model_create.restype = C.c_int
    lib.srs_model_create.argtypes = [C.POINTER(SrsSpec), C.POINTER(SrsTensor), C.c_int32,
                                     C.c_int32, C.POINTER(C.c_void_p)]
    lib.srs_model_create_ex.restype = C.c_int
    lib.srs_model_create_ex.argtypes = [C.POINTER(SrsSpec), C.POINTER(SrsTensor), C.c_int32,
                                        C.c_int32, C.c_char_p, C.POINTER(C.c_void_p)]
    lib.srs_model_destroy.restype = None
    lib.srs_model_destroy.argtypes = [C.c_void_p]
    lib.srs_predict_device.restype = C.c_int
    lib.srs_predict_device.argtypes = [C.c_void_p, C.POINTER(SrsBatch), C.c_void_p, C.c_void_p,
                                       C.c_void_p]
    lib.srs_predict_host.restype = C.c_int
    lib.srs_predict_host.argtypes = [C.c_void_p, C.POINTER(SrsBatch), C.c_void_p, C.c_void_p]
    lib.srs_predict_host_batches.restype = C.c_int
    lib.srs_predict_host_batches.argtypes = [C.c_void_p, C.c_int32, C.POINTER(SrsBatch),
                                             C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)]
    lib.srs_num_slots.restype = C.c_int
    lib.srs_predict_host_async.restype = C.c_int
    lib.srs_predict_host_async.argtypes = [C.c_void_p, C.c_int32, C.POINTER(SrsBatch), C.c_void_p,
                                           C.c_void_p]
    lib.srs_wait_slot.restype = C.c_int
    lib.srs_wait_slot.argtypes = [C.c_void_p, C.c_int32]
    lib.srs_model_status.restype = C.c_int
    lib.srs_model_status.argtypes = [C.c_void_p]
    lib.srs_model_bytes_per_inference.restype = C.c_int64
    lib.srs_model_bytes_per_inference.argtypes = [C.c_void_p]
    lib.srs_model_kernel_name.restype = C.c_char_p
    lib.srs_model_kernel_name.argtypes = [C.c_void_p]
    lib.srs_model_set_sm_limit.restype = C.c_int
    lib.srs_model_set_sm_limit.argtypes = [C.c_void_p, C.c_int32]
    lib.srs_launch_count.restype = C.c_int64
    lib.srs_fill_uniform.restype = C.c_int
    lib.srs_fill_uniform.argtypes = [C.c_void_p, C.c_int64, C.c_uint64, C.c_float, C.c_float,
                                     C.c_int32, C.c_void_p]
    lib.srs_cosine_scores_device.restype = C.c_int
    lib.srs_cosine_scores_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                             C.c_void_p, C.c_int32, C.c_void_p]
    lib.srs_topk_device.restype = C.c_int
    lib.srs_topk_device.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                    C.c_int32, C.c_void_p]
    lib.srs_rank_host.restype = C.c_int
    lib.srs_rank_host.argtypes = [C.c_void_p, C.POINTER(SrsBatch), C.c_int32, C.c_void_p,
                                  C.c_void_p]
    lib.srs_gather_create.restype = C.c_int
    lib.srs_gather_create.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int64, C.POINTER(C.c_void_p)]
    lib.srs_gather_export.restype = C.c_int
    lib.srs_gather_export.argtypes = [C.c_void_p, C.c_void_p]
    lib.srs_gather_connect.restype = C.c_int
    lib.srs_gather_connect.argtypes = [C.c_void_p, C.c_void_p]
    lib.srs_gather_destroy.restype = None
    lib.srs_gather_destroy.argtypes = [C.c_void_p]
    lib.srs_predict_device_gather.restype = C.c_int
    lib.srs_predict_device_gather.argtypes = [C.c_void_p, C.POINTER(SrsBatch), C.c_void_p, C.c_void_p]
    lib.srs_gather_wait.restype = C.c_int
    lib.srs_gather_wait.argtypes = [C.c_void_p, C.c_void_p]
    lib.srs_gather_scores.restype = C.c_int
    lib.srs_gather_scores.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int64)]
    lib.srs_gather_copy_scores.restype = C.c_int
    lib.srs_gather_copy_scores.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]
    lib.srs_model_set_movie_features.restype = C.c_int
    lib.srs_model_set_movie_features.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
    lib.srs_rank_user_host.restype = C.c_int
    lib.srs_rank_user_host.argtypes = [C.c_void_p, C.POINTER(SrsUserRow), C.c_void_p, C.c_int32, C.c_int32,
                                       C.c_void_p, C.c_void_p, C.c_void_p]
    lib.srs_selftest_wgmma.restype = C.c_int
    lib.srs_selftest_wgmma.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                      C.c_int32, C.c_int32]
    lib.srs_metrics_create.restype = C.c_int
    lib.srs_metrics_create.argtypes = [C.c_int32, C.POINTER(C.c_void_p)]
    lib.srs_metrics_destroy.restype = None
    lib.srs_metrics_destroy.argtypes = [C.c_void_p]
    lib.srs_metrics_reset.restype = C.c_int
    lib.srs_metrics_reset.argtypes = [C.c_void_p, C.c_void_p]
    lib.srs_metrics_update_device.restype = C.c_int
    lib.srs_metrics_update_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                                              C.c_void_p]
    lib.srs_metrics_update_weighted_device.restype = C.c_int
    lib.srs_metrics_update_weighted_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                       C.c_int32, C.c_void_p]
    lib.srs_metrics_result.restype = C.c_int
    lib.srs_metrics_result.argtypes = [C.c_void_p, C.POINTER(SrsEvalResult), C.c_void_p]
    lib.srs_evaluate_host_batches.restype = C.c_int
    lib.srs_evaluate_host_batches.argtypes = [C.c_void_p, C.c_int32, C.POINTER(SrsBatch), C.POINTER(C.c_void_p),
                                              C.POINTER(SrsEvalResult)]
    lib.srs_evaluate_weighted_host_batches.restype = C.c_int
    lib.srs_evaluate_weighted_host_batches.argtypes = [C.c_void_p, C.c_int32, C.POINTER(SrsBatch),
                                                       C.POINTER(C.c_void_p), C.POINTER(C.c_void_p),
                                                       C.POINTER(SrsEvalResult)]
    lib.srs_dien_outputs_device.restype = C.c_int
    lib.srs_dien_outputs_device.argtypes = [C.c_void_p, C.POINTER(SrsBatch), C.c_void_p, C.c_int32, C.c_void_p,
                                            C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.srs_dien_outputs_host_batches.restype = C.c_int
    lib.srs_dien_outputs_host_batches.argtypes = [C.c_void_p, C.c_int32, C.POINTER(SrsBatch), C.POINTER(C.c_void_p),
                                                  C.POINTER(C.c_void_p), C.POINTER(C.c_void_p),
                                                  C.POINTER(C.c_void_p)]
    lib.srs_dien_evaluate_host_batches.restype = C.c_int
    lib.srs_dien_evaluate_host_batches.argtypes = [C.c_void_p, C.c_int32, C.POINTER(SrsBatch), C.POINTER(C.c_void_p),
                                                   C.POINTER(C.c_void_p), C.POINTER(SrsDienEvalResult)]
    for f in (lib.srs_trainer_create, lib.srs_trainer_create_ex, lib.srs_trainer_create_any):
        f.restype = C.c_int
        f.argtypes = [C.POINTER(SrsSpec), C.POINTER(SrsTensor), C.c_int32, C.c_int32, C.POINTER(SrsAdam),
                      C.POINTER(C.c_void_p)]
    lib.srs_trainer_destroy.restype = None
    lib.srs_trainer_destroy.argtypes = [C.c_void_p]
    lib.srs_trainer_fit_host.restype = C.c_int
    lib.srs_trainer_fit_host.argtypes = [C.c_void_p, C.POINTER(SrsBatch), C.c_void_p, C.c_void_p, C.c_int32,
                                         C.c_int32, C.POINTER(SrsEvalResult)]
    lib.srs_trainer_get_weights.restype = C.c_int
    lib.srs_trainer_get_weights.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p]
    lib.srs_trainer_iterations.restype = C.c_int64
    lib.srs_trainer_iterations.argtypes = [C.c_void_p]
    lib.srs_trainer_fit_validate_host.restype = C.c_int
    lib.srs_trainer_fit_validate_host.argtypes = [C.c_void_p, C.POINTER(SrsBatch), C.c_void_p, C.c_void_p, C.c_int32,
                                                  C.c_int32, C.POINTER(SrsEvalResult), C.POINTER(SrsBatch),
                                                  C.c_void_p, C.c_int32, C.POINTER(SrsEvalResult)]
    lib.srs_trainer_evaluate_host.restype = C.c_int
    lib.srs_trainer_evaluate_host.argtypes = [C.c_void_p, C.POINTER(SrsBatch), C.c_void_p, C.POINTER(SrsEvalResult)]
    lib.srs_trainer_fit_weighted_host.restype = C.c_int
    lib.srs_trainer_fit_weighted_host.argtypes = [C.c_void_p, C.POINTER(SrsBatch), C.c_void_p, C.c_void_p, C.c_void_p,
                                                  C.c_int32, C.c_int32, C.POINTER(SrsEvalResult), C.POINTER(SrsBatch),
                                                  C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(SrsEvalResult)]
    lib.srs_trainer_evaluate_weighted_host.restype = C.c_int
    lib.srs_trainer_evaluate_weighted_host.argtypes = [C.c_void_p, C.POINTER(SrsBatch), C.c_void_p, C.c_void_p,
                                                       C.POINTER(SrsEvalResult)]
    lib.srs_trainer_fit_dien_host.restype = C.c_int
    lib.srs_trainer_fit_dien_host.argtypes = [C.c_void_p, C.POINTER(SrsBatch), C.c_void_p, C.c_int32, C.c_void_p,
                                              C.c_void_p, C.c_int32, C.c_int32, C.POINTER(SrsDienEvalResult)]
    lib.srs_featureeng_host.restype = C.c_int
    lib.srs_featureeng_host.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                                        C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_int32,
                                        C.POINTER(SrsSamples), C.POINTER(C.c_int64)]
    lib.srs_item2vec_host.restype = C.c_int
    lib.srs_item2vec_host.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                      C.POINTER(SrsItem2vecParams), C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                      C.POINTER(C.c_int32)]
    lib.srs_user_embeddings_host.restype = C.c_int
    lib.srs_user_embeddings_host.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int32,
                                             C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                             C.POINTER(C.c_int32)]
    lib.srs_als_fit_host.restype = C.c_int
    lib.srs_als_fit_host.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(SrsAlsParams),
                                     C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.POINTER(C.c_int32),
                                     C.c_void_p, C.c_void_p, C.POINTER(C.c_int32)]
    lib.srs_als_fit_implicit_host.restype = C.c_int
    lib.srs_als_fit_implicit_host.argtypes = lib.srs_als_fit_host.argtypes + [C.c_double]
    lib.srs_ranking_metrics_host.restype = C.c_int
    lib.srs_ranking_metrics_host.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32,
                                             C.c_int32, C.c_void_p, C.c_void_p]
    lib.srs_als_fit_folds_host.restype = C.c_int
    lib.srs_als_fit_folds_host.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32,
                                           C.c_void_p, C.c_int32, C.c_uint64, C.c_int32, C.c_int32, C.c_int32,
                                           C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.srs_als_fit_nonnegative_host.restype = C.c_int
    lib.srs_als_fit_nonnegative_host.argtypes = lib.srs_als_fit_host.argtypes + [C.c_int32, C.c_double]
    lib.srs_als_fit_folds_nonnegative_host.restype = C.c_int
    lib.srs_als_fit_folds_nonnegative_host.argtypes = lib.srs_als_fit_folds_host.argtypes + [C.c_void_p]
    lib.srs_als_recommend_host.restype = C.c_int
    lib.srs_als_recommend_host.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                           C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
    lib.srs_item_transitions_host.restype = C.c_int
    lib.srs_item_transitions_host.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32,
                                              C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                              C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int32),
                                              C.POINTER(C.c_int32)]
    lib.srs_random_walks_host.restype = C.c_int
    lib.srs_random_walks_host.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32,
                                          C.c_int32, C.c_uint64, C.c_int32, C.c_void_p, C.c_void_p]
    lib.srs_graph_embedding_host.restype = C.c_int
    lib.srs_graph_embedding_host.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                             C.POINTER(SrsItem2vecParams), C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                             C.c_void_p, C.c_void_p, C.POINTER(C.c_int32)]
    lib.srs_lsh_transform_host.restype = C.c_int
    lib.srs_lsh_transform_host.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int32, C.c_double,
                                           C.c_int32, C.c_void_p]
    lib.srs_lsh_query_host.restype = C.c_int
    lib.srs_lsh_query_host.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int32, C.c_double,
                                       C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.srs_lsh_similarity_join_host.restype = C.c_int
    lib.srs_lsh_similarity_join_host.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64,
                                                 C.c_int32, C.c_void_p, C.c_int32, C.c_double, C.c_double, C.c_int32,
                                                 C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                                                 C.POINTER(C.c_int64)]
    V, I32, I64, F64 = C.c_void_p, C.c_int32, C.c_int64, C.c_double
    lib.srs_binary_metrics_create_host.restype = C.c_int
    lib.srs_binary_metrics_create_host.argtypes = [V, V, I64, V, I32, I32, I32, C.POINTER(V)]
    lib.srs_binary_metrics_create_device.restype = C.c_int
    lib.srs_binary_metrics_create_device.argtypes = [V, V, I64, V, I32, I32, I32, V, C.POINTER(V)]
    lib.srs_binary_metrics_destroy.restype = None
    lib.srs_binary_metrics_destroy.argtypes = [V]
    lib.srs_binary_metrics_summary.restype = C.c_int
    lib.srs_binary_metrics_summary.argtypes = [V, I32, C.POINTER(SrsBinarySummary)]
    lib.srs_binary_metrics_curve.restype = C.c_int
    lib.srs_binary_metrics_curve.argtypes = [V, I32, I32, F64, V]
    lib.srs_binary_metrics_confusion.restype = C.c_int
    lib.srs_binary_metrics_confusion.argtypes = [V, I32, V, V]
    lib.srs_similar_catalog_create_host.restype = C.c_int
    lib.srs_similar_catalog_create_host.argtypes = [V, I32, V, V, I32, V, V, I64, V, V, I32, I32, I32, C.POINTER(V)]
    lib.srs_similar_catalog_destroy.restype = None
    lib.srs_similar_catalog_destroy.argtypes = [V]
    lib.srs_similar_movies_host.restype = C.c_int
    lib.srs_similar_movies_host.argtypes = [V, V, I32, I32, I32, V, V, V, V]
    lib.srs_similar_catalog_create_ex_host.restype = C.c_int
    lib.srs_similar_catalog_create_ex_host.argtypes = [V, I32, V, V, I32, V, V, I64, V, V, I32, I32, V, I32,
                                                       C.POINTER(V)]
    lib.srs_similar_movies_candidates_host.restype = C.c_int
    lib.srs_similar_movies_candidates_host.argtypes = [V, I32, V, I32, I32, I32, V, V, V, V]
    lib.srs_similar_embedding_recall_host.restype = C.c_int
    lib.srs_similar_embedding_recall_host.argtypes = [V, V, I32, I32, V, V, V, V]
    lib.srs_recforyou_users_create_host.restype = C.c_int
    lib.srs_recforyou_users_create_host.argtypes = [V, I64, V, V, I32, I32, I32, C.POINTER(V)]
    lib.srs_recforyou_users_destroy.restype = None
    lib.srs_recforyou_users_destroy.argtypes = [V]
    lib.srs_recforyou_host.restype = C.c_int
    lib.srs_recforyou_host.argtypes = [V, V, V, I32, V, I32, I32, V, V, V, V]
    lib.srs_recforyou_users_set_features_host.restype = C.c_int
    lib.srs_recforyou_users_set_features_host.argtypes = [V, I32, V, V, V, V]
    lib.srs_recforyou_ctr_host.restype = C.c_int
    lib.srs_recforyou_ctr_host.argtypes = [V, V, V, V, I32, I32, V, V, V, V]
    for name, args in (
            ("srs_approx_quantile_host", [V, I64, V, I32, F64, I32, V]),
            ("srs_quantile_discretizer_host", [V, I64, I32, F64, I32, V, C.POINTER(I32), V]),
            ("srs_bucketize_host", [V, I32, V, I64, I32, V]),
            ("srs_minmax_scale_host", [V, I64, V, I32, V, V]),
            ("srs_rating_features_host", [V, V, I64, I32, I32, V, V, V, V, C.POINTER(I32)]),
            ("srs_string_indexer_host", [V, I64, V, I32, I32, V, V]),
            ("srs_genre_multihot_host", [V, V, V, I32, V, I32, I32, V, V, V, V, V]),
            ("srs_sample_split_host", [I64, C.c_uint64, F64, V, I32, I32, V, V]),
            ("srs_sample_split_by_timestamp_host", [V, I64, C.c_uint64, F64, F64, I32, V, V, C.POINTER(F64)])):
        f = getattr(lib, name)
        f.restype = C.c_int
        f.argtypes = args
    if lib.srs_abi_version() != ABI_VERSION:
        raise ImportError("libsrs_ctr.so ABI version %d != %d" % (lib.srs_abi_version(), ABI_VERSION))
    _lib = lib
    return lib


def check(rc: int):
    if rc == SRS_OK:
        return
    msg = load().srs_last_error().decode("utf-8", "replace")
    if rc == SRS_ERR_RANGE:
        raise ValueError(msg)            # mirrors TF's assert on identity columns
    if rc == SRS_ERR_MISSING:
        raise KeyError(msg)
    if rc == SRS_ERR_INVALID:
        raise SrsInvalidError(rc, msg)
    raise SrsError(rc, msg)
