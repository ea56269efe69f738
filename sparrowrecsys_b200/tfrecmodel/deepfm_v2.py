"""tfrecmodel.deepfm_v2 - H100 drop-in for the reference's `DeepFM_v2.py` model
(TFRecModel/src/com/sparrowrecsys/offline/tensorflow/DeepFM_v2.py:98-173).

    from tfrecmodel import deepfm_v2
    deepfm_v2.load(weights)            # or load(savedmodel=...), load(spec=..., seed=...)
    p = deepfm_v2.predict(features)    # dict of 1-D columns -> float32 [N,1]
    loss, acc, roc_auc, pr_auc = deepfm_v2.evaluate(test_features)   # rows labelled by "label"
    history = deepfm_v2.fit(train_features, epochs=5)   # rebuilds `model` from the result
"""
from ._surface import Surface

_surface = Surface("deepfm_v2")
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


def fit(features, epochs=5, batch_size=12, seed=0, validation_data=None, validation_split=0.0, validation_freq=1,
        sample_weight=None, class_weight=None):
    """`model.fit(train_dataset, epochs=5)` (DeepFM_v2.py:165): train from the loaded weights on the GPU, then rebuild
    `model` from the trained weights; returns Keras's history dict {"loss", "accuracy", "auc", "auc_1"} (one value
    per epoch), plus "val_loss", "val_accuracy", "val_auc", "val_auc_1" for the validated epochs when
    `validation_data` or `validation_split` is given (`Trainer.fit`)."""
    global model
    history = _surface.fit(features, epochs, batch_size, seed, validation_data, validation_split, validation_freq,
                           sample_weight, class_weight)
    model = _surface.model
    return history
