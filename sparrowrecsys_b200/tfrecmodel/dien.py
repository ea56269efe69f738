"""tfrecmodel.dien - H100 drop-in for the reference's `DIEN.py` model
(TFRecModel/src/com/sparrowrecsys/offline/tensorflow/DIEN.py:154-296), with the AUGRU's initial state a
stored weight (`augru_h0`) instead of a fresh random draw per call (:235-236).

    from tfrecmodel import dien
    dien.load(weights)            # or load(savedmodel=...), load(spec=..., seed=...)
    p = dien.predict(features)    # dict of 1-D columns -> float32 [N,1] (y_pred)
    y_pred, final_loss = dien.predict_outputs(features, batch_size=12)   # model.predict, both outputs (:312)
    dien.evaluate_outputs(features, batch_size=12)   # model.evaluate (:304) -> {"loss", "auc", "auc_value"}
    history = dien.fit(train_features, epochs=5)     # model.fit (:300), in file order; rebuilds `model`

The two-output calls and `fit` need the auxiliary-head weights (`weights.init_aux_weights`) and the inputs
`negtive_userRatedMovie2..5` (`features.negative_history`) and `label`.
"""
from ..weights import init_aux_weights, init_weights
from ._surface import Surface

_surface = Surface("dien")
model = None          # the module-level model, as in the reference script
spec = _surface.spec


def load(weights=None, spec=None, seed=None, savedmodel=None, device=0):
    """As the other modules; an untrained model (no `weights`) also gets the auxiliary head's initial
    weights, as the reference's `model` holds them before fit."""
    global model
    if weights is None and savedmodel is None:
        sp = spec or _surface.spec()
        s = 0 if seed is None else seed
        weights = {**init_weights(sp, s, for_test=False), **init_aux_weights(sp, s)}
    model = _surface.load(weights, spec, seed, savedmodel, device)
    return model


def predict(features, batch_size=None):
    return _surface.predict(features, batch_size)


def predict_outputs(features, batch_size=None):
    """`model.predict(test_dataset)` of the two-output model (DIEN.py:312): [y_pred [N,1], final_loss [N]]."""
    if _surface.model is None:
        raise RuntimeError("tfrecmodel.dien: call load() before predict_outputs()")
    return _surface.model.dien_outputs(features, batch_size)


def evaluate_outputs(features, batch_size=None):
    """`model.evaluate(test_dataset)` of the reference's DIEN (DIEN.py:304): {"loss", "auc", "auc_value"}."""
    if _surface.model is None:
        raise RuntimeError("tfrecmodel.dien: call load() before evaluate_outputs()")
    return _surface.model.dien_evaluate(features, batch_size)


def evaluate(features, batch_size=None):
    """Not this call: the other modules' `evaluate` reports the four compile metrics (loss, accuracy, roc_auc,
    pr_auc), which DIEN's script never compiles.  Its `model.evaluate` reports the loss with the auxiliary
    negative-sample term and the layer's AUC metrics: that is `evaluate_outputs`."""
    raise NotImplementedError("tfrecmodel.dien.evaluate: DIEN's Keras evaluate reports the loss with the auxiliary "
                              "negative-sample term and its AUC metrics, not the four compile metrics; use "
                              "tfrecmodel.dien.evaluate_outputs (CTRModel.dien_evaluate)")


def fit(features, epochs=5, batch_size=12, seed=0):
    """`model.fit(train_dataset, epochs=5)` (DIEN.py:300): train from the loaded weights on the GPU, in file order
    every epoch (the script's dataset has no shuffle; `seed` is not used), then rebuild `model` from the trained
    weights; returns the history dict {"loss", "auc", "auc_value"} (one value per epoch).  `features` also carries
    `negtive_userRatedMovie2..5` and `label`, as for `evaluate_outputs`."""
    global model
    history = _surface.fit(features, epochs, batch_size, seed)
    model = _surface.model
    return history
