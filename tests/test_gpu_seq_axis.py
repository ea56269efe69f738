"""The history axis of the sequence kernels on the GPU: every `SEQ_MATRIX` case of tests/test_seq_axis.py runs its
kernel, matches the float64 oracle and repeats bit for bit (needs a GPU: pytest -m gpu).

The cases past 2^24 build a table of 2^24 + 4 movies with srs_fill_uniform on the device (lent to the model as it is
at E = 32, copied to the host for E = 10, whose rows the model pads to 12).  The oracle regenerates only the rows a
batch touches.  Past 2^24 each case also holds that the id 2^24 + 3, in range as given but not after its float32
rounding, is an error: in a served batch it latches the range error and every other row scores as without it; in
`fit` it is rejected before any launch, in the candidate, the history or the negatives, and nothing changes."""
import numpy as np
import pytest

import test_dien_aux
from oracle import dien_train
from sparrowrecsys_b200.features import encode_batch, negative_history_keys
from sparrowrecsys_b200.spec import history_keys
from test_seq_axis import (AUX_ATOL, AUX_RTOL, BIG_VOCAB, FIT_BATCH, FIT_CASES, FORWARD_CASES, PROB_ATOL,
                           ROUNDS_OUT, TABLE_HI, TABLE_LO, TABLE_SEED, _ids, aux_oracle, compact, features,
                           logit_atol, oracle, past_2_24, row0, spec_of, touched_rows, weights)

pytestmark = pytest.mark.gpu

BAD_ROW = 11                    # the row that carries 2^24 + 3 in the error checks


def _device_used(label):
    """Print the device memory in use (every process's; the machine may be shared) beside `label`."""
    import torch
    free, total = torch.cuda.mem_get_info(0)
    print("device memory in use %s: %.2f GB" % (label, (total - free) / 1e9))


def _big_table(E):
    """The [2^24 + 4][E] behaviour table of test_seq_axis.big_table_rows, generated in HBM."""
    import torch
    from sparrowrecsys_b200 import _lib
    t = torch.empty(BIG_VOCAB, E, dtype=torch.float32, device="cuda:0")
    _lib.check(_lib.load().srs_fill_uniform(t.data_ptr(), t.numel(), TABLE_SEED, TABLE_LO, TABLE_HI, 0, None))
    t[0] = torch.from_numpy(row0(E)).cuda()
    torch.cuda.synchronize()
    return t


def _with_table(case, W):
    """The case's weights with its behaviour table: the device table past 2^24 (lent to the model when E is
    already a padded width, a host copy otherwise)."""
    import torch
    if not past_2_24(case):
        return W
    t = _big_table(case.E)
    if case.E in (12, 16, 32, 64):
        return dict(W, embedding=t)
    host = t.cpu().numpy()
    del t
    torch.cuda.empty_cache()
    return dict(W, embedding=host)


def _model(case, W):
    from sparrowrecsys_b200.model import CTRModel
    return CTRModel(spec_of(case), W, device=0, options={"din_impl": case.impl} if case.impl else None)


def _negatives(case, f):
    import torch
    T = case.T
    neg = np.stack([np.asarray(f[k], np.int32) for k in negative_history_keys(T)], 1) if T > 1 \
        else np.zeros((case.B, 0), np.int32)
    return torch.from_numpy(np.ascontiguousarray(neg)).cuda()


def _run(case, m, enc, f, expect_error=False):
    """(probs, logits[, aux, final_loss]) of one device launch of the case's kernel over the encoded batch."""
    import torch
    dev = m.to_device(enc)
    if case.aux:
        lab = torch.from_numpy(np.asarray(f["label"], np.int32)).cuda()
        out = [torch.empty(case.B, dtype=torch.float32, device="cuda:0") for _ in range(4)]
        test_dien_aux._dien_device(m, dev, _negatives(case, f), max(case.T - 1, 0), lab, *out)
    else:
        out = [torch.empty(case.B, dtype=torch.float32, device="cuda:0") for _ in range(2)]
        m.predict_device(dev, out[0], out[1])
    if expect_error:
        with pytest.raises(ValueError):
            m.status()
    m.status()
    return [t.cpu().numpy() for t in out]


def _check(case, W, f, got):
    po, zo = oracle(case, W, f)
    p, z = got[0], got[1]
    print(case.name, "logit err %.3g prob err %.3g" % (np.abs(z - zo[:, 0]).max(), np.abs(p - po[:, 0]).max()))
    assert np.abs(z - zo[:, 0]).max() <= logit_atol(case), "logit err %g" % np.abs(z - zo[:, 0]).max()
    assert np.abs(p - po[:, 0]).max() <= PROB_ATOL, "prob err %g" % np.abs(p - po[:, 0]).max()
    if case.aux:
        aux, fl = got[2], got[3]
        want = aux_oracle(case, W, f)
        print(case.name, "aux err %.3g" % np.abs(aux - want).max())
        assert np.allclose(aux, want, rtol=AUX_RTOL, atol=AUX_ATOL), np.abs(aux - want).max()
        # final_loss_i = bce_i - 0.5 * mean(aux): it carries the tolerance of the aux mean
        fl_want = test_dien_aux.final_loss_oracle(z, f["label"], want)
        fl_atol = 1e-5 + 0.5 * AUX_RTOL * np.abs(want).mean()
        assert np.abs(fl - fl_want).max() <= fl_atol, np.abs(fl - fl_want).max()


@pytest.mark.parametrize("case", FORWARD_CASES, ids=_ids)
def test_case_matches_the_float64_oracle(case):
    W, f = weights(case), features(case)
    Wd = _with_table(case, W)
    enc = encode_batch(spec_of(case), f)
    with _model(case, Wd) as m:
        assert m.kernel_name == case.kernel
        if past_2_24(case):
            _device_used("while %s is served" % case.name)
        got = _run(case, m, enc, f)
        again = _run(case, m, f=f, enc=enc)
        assert all(np.array_equal(a, b) for a, b in zip(got, again))     # a second run gives the same bits
        if not case.aux:                                                  # the host path gives the same bits
            p, z = m.predict_with_logits(f)
            assert np.array_equal(p[:, 0], got[0]) and np.array_equal(z[:, 0], got[1])
        if past_2_24(case):
            # 2^24 + 3 in one row's history: the range error latches, the other rows keep their bits
            bad = encode_batch(spec_of(case), f)
            bad.hist = bad.hist.copy()
            bad.hist[BAD_ROW, case.T // 2] = ROUNDS_OUT
            err = _run(case, m, bad, f, expect_error=True)
            keep = np.arange(case.B) != BAD_ROW
            for a, b in zip(err[:3], got[:3]):                            # probs, logits, aux
                assert np.array_equal(a[keep], b[keep])
            assert all(np.array_equal(a, b) for a, b in zip(_run(case, m, enc, f), got))
    _check(case, W, f, got)


@pytest.mark.parametrize("case", FIT_CASES, ids=_ids)
def test_fit_past_2_24(case):
    """DIEN's fit on a table of 2^24 + 4 rows: 2^24 + 3 anywhere is rejected before any launch and changes nothing;
    then one epoch in steps of FIT_BATCH matches the float64 oracle on the touched rows (the float32-spread rule of
    test_gpu_fit_dien.py), and every other row keeps its bits: a row whose Adam moments stay 0 does not move."""
    from sparrowrecsys_b200.model import launch_count
    from sparrowrecsys_b200.training import Trainer
    from test_gpu_fit_dien import _check_close
    W, f = weights(case), features(case)
    Wd = _with_table(case, W)
    T = case.T
    with Trainer(spec_of(case), Wd) as tr:
        _device_used("while %s trains" % case.name)
        for key in ("movieId", history_keys(T)[T // 2], negative_history_keys(T)[1]):
            bad = dict(f)
            bad[key] = np.array(f[key], copy=True)
            bad[key][BAD_ROW] = ROUNDS_OUT
            before = launch_count()
            with pytest.raises(ValueError, match=str(ROUNDS_OUT)):
                tr.fit(bad, epochs=1, batch_size=FIT_BATCH)
            assert launch_count() == before, key
        assert tr.iterations == 0
        now = tr.weights()
        assert all(np.array_equal(now[k], Wd[k]) for k in Wd)
        del now
        tr.fit(f, epochs=1, batch_size=FIT_BATCH)
        assert tr.iterations == -(-case.B // FIT_BATCH)
        got = tr.weights()
    touched = touched_rows(case, f)
    untouched = np.ones(BIG_VOCAB, bool)
    untouched[touched] = False
    assert np.array_equal(got["embedding"][untouched], Wd["embedding"][untouched])
    spec_c, Wc, fc = compact(case, f, W)
    rows = dien_train.Rows.from_features(fc, T)
    w64, _, _ = dien_train.fit(Wc, rows, [np.arange(case.B)], FIT_BATCH, np.float64)
    w32, _, _ = dien_train.fit(Wc, rows, [np.arange(case.B)], FIT_BATCH, np.float32)
    assert np.array_equal(Wc["embedding"], Wd["embedding"][touched])
    _check_close(dict(got, embedding=got["embedding"][touched]), w64, w32, case.name)
