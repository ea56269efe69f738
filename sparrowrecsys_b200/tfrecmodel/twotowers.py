"""tfrecmodel.twotowers - H100 drop-in for the reference's `NeuralCF.py` model
(TFRecModel/src/com/sparrowrecsys/offline/tensorflow/NeuralCF.py:57-70).

    from tfrecmodel import twotowers
    twotowers.load(weights)            # or load(savedmodel=...), load(spec=..., seed=...)
    p = twotowers.predict(features)    # dict of 1-D columns -> float32 [N,1]
    loss, acc, roc_auc, pr_auc = twotowers.evaluate(test_features)   # rows labelled by "label"
"""
from ._surface import Surface

_surface = Surface("twotowers")
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
    """Not part of this surface: the `tfrecmodel.<name>.fit` calls restate each script's own `model.fit`, and
    NeuralCF.py fits only its first model, neural_cf_model_1 (`tfrecmodel.neuralcf.fit`).  The two-tower model trains
    on the GPU through `sparrowrecsys_b200.training.Trainer` (with its final Dense; DESIGN.md section 4.27)."""
    raise NotImplementedError("tfrecmodel.twotowers: NeuralCF.py fits only neural_cf_model_1 (tfrecmodel.neuralcf."
                              "fit); train the two-tower model with sparrowrecsys_b200.training.Trainer")
