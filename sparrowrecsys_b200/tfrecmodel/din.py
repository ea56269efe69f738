"""tfrecmodel.din - H100 drop-in for the reference's `DIN.py` model
(TFRecModel/src/com/sparrowrecsys/offline/tensorflow/DIN.py:125-185).

    from tfrecmodel import din
    din.load(weights)            # or load(savedmodel=...), load(spec=..., seed=...)
    p = din.predict(features)    # dict of 1-D columns -> float32 [N,1]
    loss, acc, roc_auc, pr_auc = din.evaluate(test_features)   # rows labelled by "label"
"""
from ._surface import Surface

_surface = Surface("din")
model = None          # the module-level model, as in the reference script
spec = _surface.spec


def load(weights=None, spec=None, seed=None, savedmodel=None, device=0):
    global model
    model = _surface.load(weights, spec, seed, savedmodel, device)
    return model


def predict(features, batch_size=None):
    return _surface.predict(features, batch_size)


def evaluate(features, batch_size=None, sample_weight=None):
    """`model.evaluate(x, sample_weight=...)`: (loss, accuracy, roc_auc, pr_auc), weighted when given."""
    return _surface.evaluate(features, batch_size, sample_weight)


def fit(features, epochs=5, batch_size=12, seed=0):
    """Not implemented for this model: `fit` covers NeuralCF (tfrecmodel.neuralcf) and DeepFM (tfrecmodel.deepfm)
    only."""
    return _surface.fit(features, epochs, batch_size, seed)
