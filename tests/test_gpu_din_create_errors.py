"""DIN model creation with a missing or misshapen weight tensor (needs a GPU: pytest -m gpu).

`CTRModel` checks the weights in Python before the C call, so these tests hand the tensors to
`srs_model_create` through `_lib` directly: the library's own lookup must name the tensor and return
SRS_ERR_MISSING / SRS_ERR_SHAPE, and with two tensors missing it reports the first one it looks up
(the four tables, then au_dense/kernel .. dense_2/bias)."""
import ctypes as C

import numpy as np
import pytest

from sparrowrecsys_b200 import _lib
from sparrowrecsys_b200.model import _spec_struct
from sparrowrecsys_b200.spec import default_spec
from sparrowrecsys_b200.weights import init_weights, weight_shapes

pytestmark = pytest.mark.gpu

SPEC = default_spec("din", emb_dim=32, hist_len=20, n_movies=3000, n_users=2000)
CHECKED = ["embedding", "au_dense/kernel", "au_prelu/alpha", "dense/kernel", "prelu_1/alpha"]


def _create(weights, shapes=None):
    """srs_model_create on `weights` (name -> host array); `shapes` overrides a tensor's declared
    [rows, cols].  Returns (return code, srs_last_error())."""
    lib = _lib.load()
    keep = []
    tensors = (_lib.SrsTensor * len(weights))()
    for i, (name, w) in enumerate(weights.items()):
        a = np.ascontiguousarray(w, dtype=np.float32)
        keep.append(a)
        rows, cols = (shapes or {}).get(name, (a.shape[0], a.shape[1] if a.ndim > 1 else 1))
        tensors[i] = _lib.SrsTensor(name.encode(), a.ctypes.data, rows, cols, _lib.SRS_HOST)
    out = C.c_void_p()
    rc = lib.srs_model_create(C.byref(_spec_struct(SPEC)), tensors, len(weights), 0, C.byref(out))
    err = lib.srs_last_error().decode()
    if out.value:
        lib.srs_model_destroy(out)
    return rc, err


def test_din_weights_as_given_create_a_model():
    rc, err = _create(init_weights(SPEC, 1))
    assert rc == _lib.SRS_OK, err


@pytest.mark.parametrize("name", CHECKED)
def test_din_create_names_a_missing_tensor(name):
    W = init_weights(SPEC, 1)
    del W[name]
    rc, err = _create(W)
    assert rc == _lib.SRS_ERR_MISSING
    assert err == "missing weight tensor '%s'" % name


@pytest.mark.parametrize("name", CHECKED)
def test_din_create_names_a_misshapen_tensor(name):
    W = init_weights(SPEC, 1)
    shape = dict(weight_shapes(SPEC))[name]
    rows, cols = shape[0], shape[1] if len(shape) > 1 else 1
    W[name] = np.zeros((rows + 1, cols), np.float32)
    rc, err = _create(W)
    assert rc == _lib.SRS_ERR_SHAPE
    assert err == "weight '%s' has shape [%d,%d], expected [%d,%d]" % (name, rows + 1, cols, rows, cols)


@pytest.mark.parametrize("first,second", [("embedding", "dense/kernel"), ("au_dense/kernel", "au_prelu/alpha"),
                                          ("au_prelu/alpha", "prelu_1/alpha"), ("dense/kernel", "prelu_1/alpha")])
def test_din_create_reports_the_first_missing_tensor_in_lookup_order(first, second):
    W = init_weights(SPEC, 1)
    # both dropped, and the caller's list reversed: the library's lookup order decides, not the list's
    W = {k: W[k] for k in reversed(list(W)) if k not in (first, second)}
    rc, err = _create(W)
    assert rc == _lib.SRS_ERR_MISSING
    assert err == "missing weight tensor '%s'" % first
