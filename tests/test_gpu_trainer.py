"""GPU checks of the trainer every model shares (csrc/trainer.cu, DESIGN.md sections 4.8-4.10 and 4.18-4.20): the
launches of a fit, per step, per epoch and per validated epoch, and a trainer on a second device after a fit on the
first (the step kernels' dynamic shared memory opt-in is per device)."""
import numpy as np
import pytest

from sparrowrecsys_b200.spec import default_spec
from sparrowrecsys_b200.weights import init_aux_weights, init_weights

MODELS = ["neuralcf", "deepfm", "widendeep", "deepfm_v2", "dien"]
# launches per step and per epoch (the table at the top of csrc/trainer.cu); a validated epoch adds 2
PER_STEP = {"neuralcf": 5, "deepfm": 7, "widendeep": 7, "deepfm_v2": 7, "dien": 6}
PER_EPOCH = {"neuralcf": 0, "deepfm": 1, "widendeep": 1, "deepfm_v2": 1, "dien": 3}
# the largest embedding width of each model: every step at it asks for more than 48 KiB of shared memory (NeuralCF's
# at three 32-wide hidden layers)
LARGE = {"neuralcf": dict(emb_dim=64, hidden=(32, 32, 32)), "deepfm": dict(emb_dim=64),
         "widendeep": dict(emb_dim=64), "deepfm_v2": dict(emb_dim=64), "dien": dict(emb_dim=32)}


def _setup(model, n, **over):
    from sparrowrecsys_b200.features import negative_history, synthetic_features
    spec = default_spec(model, **over)
    W = init_weights(spec, 0)
    if model == "dien":
        W.update(init_aux_weights(spec, 0))
    f = synthetic_features(spec, n, seed=3)
    if model == "dien":
        f.update(negative_history(f, spec.hist_len, 3, n_movies=spec.n_movies))
    f["label"] = (np.random.default_rng(3).random(n) < 0.4).astype(np.int32)
    return spec, W, f


@pytest.mark.gpu
@pytest.mark.parametrize("model", MODELS)
def test_launches_per_step_epoch_and_validated_epoch(model):
    from sparrowrecsys_b200.model import launch_count
    from sparrowrecsys_b200.training import Trainer
    spec, W, f = _setup(model, 30)
    epochs, steps = 2, 3                               # batches of 12, 12 and 6
    with Trainer(spec, W) as tr:
        n0 = launch_count()
        tr.fit(f, epochs=epochs, batch_size=12)
        assert launch_count() - n0 == epochs * (steps * PER_STEP[model] + PER_EPOCH[model])
        if model == "dien":
            return
        n0 = launch_count()
        tr.fit(f, epochs=epochs, batch_size=12, validation_data=f)
        assert launch_count() - n0 == epochs * (steps * PER_STEP[model] + PER_EPOCH[model] + 2)


@pytest.mark.gpu
@pytest.mark.parametrize("model", MODELS)
def test_a_second_device_fits_what_the_first_fits(model):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs on the box")
    from sparrowrecsys_b200.training import Trainer
    spec, W, f = _setup(model, 100, **LARGE[model])
    out = []
    for device in (0, 1):
        with Trainer(spec, W, device=device) as tr:
            hist = tr.fit(f, epochs=2, batch_size=33)
            out.append((hist, tr.weights(), tr.iterations))
    (h0, w0, it0), (h1, w1, it1) = out
    assert h0 == h1 and it0 == it1
    assert w0.keys() == w1.keys()
    for k in w0:
        assert np.array_equal(w0[k], w1[k]), k
