"""Shared implementation of the per-model `tfrecmodel.<name>` modules.

Each reference model script is a flat module whose public surface is the
module-level Keras `model` and the call `model.predict(feature_dict)`
(`TFRecModel/src/com/sparrowrecsys/offline/tensorflow/<Name>.py`).  The modules in
this package keep that surface: `load(...)` builds the module-level `model` (a
`sparrowrecsys_b200.model.CTRModel` living on one GPU), `predict(features)` is
`model.predict(features)` and `evaluate(features)` is `model.evaluate(test_dataset)`, the last
call of each script (e.g. DIN.py:171-185).
"""
from __future__ import annotations

from typing import Mapping, Optional

import numpy as np

from ..model import CTRModel
from ..spec import ModelSpec, default_spec
from ..weights import init_weights


class Surface:
    def __init__(self, name: str):
        self.name = name
        self.model: Optional[CTRModel] = None
        self.weights = None       # the host weights `model` was built from (None: a shipped export of another model)

    def spec(self, **overrides) -> ModelSpec:
        """The reference script's own constants unless overridden."""
        return default_spec(self.name, **overrides)

    def load(self, weights: Optional[Mapping[str, np.ndarray]] = None,
             spec: Optional[ModelSpec] = None, seed: Optional[int] = None,
             savedmodel: Optional[str] = None, device: int = 0) -> CTRModel:
        if self.model is not None:
            self.model.close()
            self.model = None
        self.weights = None
        if savedmodel is not None:
            if self.name == "neuralcf":                 # kept on the host, so that fit() can start from them
                from ..bundle import load_neuralcf
                self.weights = load_neuralcf(savedmodel)
                self.model = CTRModel(default_spec("neuralcf"), self.weights, device)
            else:
                self.model = CTRModel.from_savedmodel(savedmodel, self.name, device)
            return self.model
        spec = spec or self.spec()
        if spec.model != self.name:
            raise ValueError("spec is for %r, this module is %r" % (spec.model, self.name))
        if weights is None:
            # untrained model: the reference's initialisers (what `model` holds before fit)
            weights = init_weights(spec, 0 if seed is None else seed, for_test=False)
        self.model = CTRModel(spec, weights, device)
        self.weights = weights
        return self.model

    def predict(self, features, batch_size: Optional[int] = None) -> np.ndarray:
        if self.model is None:
            raise RuntimeError("tfrecmodel.%s: call load() before predict()" % self.name)
        return self.model.predict(features, batch_size)

    def evaluate(self, features, batch_size: Optional[int] = None, sample_weight=None):
        """(loss, accuracy, roc_auc, pr_auc) over the labelled rows (`features["label"]`), weighted by
        `sample_weight` when given."""
        if self.model is None:
            raise RuntimeError("tfrecmodel.%s: call load() before evaluate()" % self.name)
        if sample_weight is None:
            return self.model.evaluate(features, batch_size=batch_size)
        return self.model.evaluate(features, batch_size=batch_size, sample_weight=sample_weight)

    def fit(self, features, epochs: int = 5, batch_size: int = 12, seed: int = 0, validation_data=None,
            validation_split: float = 0.0, validation_freq: int = 1, sample_weight=None,
            class_weight=None) -> dict:
        """`model.fit(train_dataset, epochs=5)` (NeuralCF.py:91, DeepFM.py, WideNDeep.py:117,
        DeepFM_v2.py:165): train from the weights `model` was loaded with, then rebuild `model` from the trained
        weights.  Returns Keras's history dict, with the `val_*` lists when `validation_data` or
        `validation_split` is given (`Trainer.fit`).  NeuralCF, DeepFM, Wide&Deep, DeepFM_v2 and DIEN only (DIEN: in
        file order, without validation, its history {"loss", "auc", "auc_value"})."""
        if self.name not in ("neuralcf", "deepfm", "widendeep", "deepfm_v2", "dien"):
            raise NotImplementedError("tfrecmodel.%s: fit is implemented for NeuralCF (tfrecmodel.neuralcf), "
                                      "DeepFM (tfrecmodel.deepfm), Wide&Deep (tfrecmodel.widendeep), DeepFM_v2 "
                                      "(tfrecmodel.deepfm_v2) and DIEN (tfrecmodel.dien) only" % self.name)
        if self.model is None or self.weights is None:
            raise RuntimeError("tfrecmodel.%s: call load() before fit()" % self.name)
        from ..training import Trainer
        spec, device = self.model.spec, self.model.device
        with Trainer(spec, self.weights, device) as tr:
            weighting = {} if sample_weight is None and class_weight is None else \
                {"sample_weight": sample_weight, "class_weight": class_weight}
            history = tr.fit(features, epochs=epochs, batch_size=batch_size, seed=seed,
                             validation_data=validation_data, validation_split=validation_split,
                             validation_freq=validation_freq, **weighting)
            trained = tr.weights()
        self.model.close()
        self.model = CTRModel(spec, trained, device)
        self.weights = trained
        return history
