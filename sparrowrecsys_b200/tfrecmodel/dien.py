"""tfrecmodel.dien - H100 drop-in for the forward pass (`y_pred`) of the reference's `DIEN.py`
model (TFRecModel/src/com/sparrowrecsys/offline/tensorflow/DIEN.py:154-256), with the AUGRU's
initial state a stored weight (`augru_h0`) instead of a fresh random draw per call (:235-236).

    from tfrecmodel import dien
    dien.load(weights)            # or load(savedmodel=...), load(spec=..., seed=...)
    p = dien.predict(features)    # dict of 1-D columns -> float32 [N,1]
"""
from ._surface import Surface

_surface = Surface("dien")
model = None          # the module-level model, as in the reference script
spec = _surface.spec


def load(weights=None, spec=None, seed=None, savedmodel=None, device=0):
    global model
    model = _surface.load(weights, spec, seed, savedmodel, device)
    return model


def predict(features, batch_size=None):
    return _surface.predict(features, batch_size)


def evaluate(features, batch_size=None):
    """Not covered: the reference's DIEN `model.evaluate` returns (loss, roc_auc) with a loss that includes
    the auxiliary negative-sample loss (DIEN.py:261-304), which is training-only and not computed here."""
    raise NotImplementedError("tfrecmodel.dien.evaluate: DIEN's Keras evaluate loss includes the auxiliary "
                              "negative-sample loss, which is training-only and not computed by this library")
