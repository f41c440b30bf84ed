"""The engine-arithmetic emulation (folded order, fp16/bf16 operand rounding) against the
reference-order oracle.  States the FP tolerance of the product path on the CPU."""
import numpy as np
import pytest
import torch

import helpers
import kernel_jobs as K
from oracle import contract as C
from oracle import wavernn_oracle as O


@pytest.fixture(scope="module")
def setup():
    model = helpers.make_model(0, "MOL")
    sd = helpers.state_numpy(model)
    w = O.hot_weights(sd)
    mel_p = O.pad_time(helpers.make_mel(30, 0)[0].numpy().T, 2).T
    m_up, aux = O.upsample_network(sd, mel_p, pad=2)
    U = helpers.replay_uniforms(1234, 3300, 3)
    kw = dict(n_seg=3, seg_len=3300, seg_stride=3025, uniforms=U, steps=400)
    ref, lref = O.generate_segments(w, m_up, aux, want_logits=True, **kw)
    return w, m_up, aux, kw, ref, lref


def test_rounders():
    x = np.array([1.0, 1.00390625, 1.001953125, 65504.0, 1e6, -1e6, 3e-8, 0.1], np.float32)
    assert C.bf16_round(x)[1] == np.float32(1.0)                    # tie to even
    assert C.fp16_round(x)[4] == np.float32(65504.0) and C.fp16_round(x)[5] == np.float32(-65504.0)
    assert abs(C.fp16_round(x)[7] - 0.1) < 1e-4 and abs(C.bf16_round(x)[7] - 0.1) < 1e-3


def test_folded_fp32_equals_reference_order(setup):
    w, m_up, aux, kw, ref, lref = setup
    out, lg = C.generate_segments(w, m_up, aux, precision="fp32", want_logits=True, **kw)
    np.testing.assert_allclose(lg, lref, rtol=0, atol=2e-5)
    np.testing.assert_allclose(out, ref, rtol=0, atol=2e-5)


@pytest.mark.parametrize("precision,tol", [("fp16", 2e-3), ("bf16", 1.5e-2)])
def test_operand_rounding_teacher_forced_tolerance(setup, precision, tol):
    """Teacher-forced (reference samples fed back): per-step logits of the rounded-operand
    arithmetic stay within `tol` of the fp32 reference for this model."""
    w, m_up, aux, kw, ref, lref = setup
    _, lg = C.generate_segments(w, m_up, aux, precision=precision, want_logits=True, x_force=ref.T.copy(), **kw)
    assert np.abs(lg - lref).max() < tol


def test_fold_tables_of_the_strided_windows_reproduce_the_strided_run_and_short_windows_read_zero_rows(setup):
    w, m_up, aux, kw, _, _ = setup
    kw = dict(kw, steps=40)
    B, stride, L = kw["n_seg"], kw["seg_stride"], m_up.shape[0]
    base = np.arange(B, dtype=np.int64) * stride
    out, lg = C.generate_segments(w, m_up, aux, want_logits=True, **kw)
    out_t, lg_t = C.generate_segments(w, m_up, aux, want_logits=True, fold_row0=base, fold_row_end=np.full(B, L), **kw)
    assert np.array_equal(out, out_t) and np.array_equal(lg, lg_t)
    # windows of 25, 1 and 40 rows: the same as the strided run on rows zeroed past each window's end
    end = base + np.array([25, 1, 40])
    m_z, a_z = m_up.copy(), aux.copy()
    for f in range(B):
        m_z[end[f]:base[f] + 40] = 0
        a_z[end[f]:base[f] + 40] = 0
    out_z, lg_z = C.generate_segments(w, m_z, a_z, want_logits=True, **kw)
    out_e, lg_e = C.generate_segments(w, m_up, aux, want_logits=True, fold_row0=base, fold_row_end=end, **kw)
    assert np.array_equal(out_z, out_e) and np.array_equal(lg_z, lg_e)
    assert not np.array_equal(lg_e, lg)


def test_expand_rows_restates_the_upsample_network():
    """contract.expand_rows (float64 5-tap sum over the padded mel) against model.upsample, the whole stream and a
    slice starting at a non-zero phase."""
    model = helpers.make_model(0, "MOL").eval()
    T, hop = 23, 275
    mp = torch.nn.functional.pad(helpers.make_mel(T, 4), (2, 2))
    with torch.no_grad():
        full_m, full_a = model.upsample(mp)
        aux_fr = model.upsample.resnet(mp)[0].T.numpy()
    taps = model.upsample_taps(torch.device("cpu")).numpy()
    mel_fr = mp[0].T.numpy()
    m, a = C.expand_rows(mel_fr, aux_fr, taps, hop, 0, T * hop)
    np.testing.assert_allclose(m, full_m[0].numpy(), rtol=0, atol=2e-6)
    assert np.array_equal(a, full_a[0].numpy())
    m2, a2 = C.expand_rows(mel_fr, aux_fr, taps, hop, 3 * hop + 101, 700)
    assert np.array_equal(m2, m[3 * hop + 101:3 * hop + 801]) and np.array_equal(a2, a[3 * hop + 101:3 * hop + 801])


@pytest.mark.parametrize("precision", ["fp16", "bf16"])
@pytest.mark.parametrize("mode", ["MOL", "RAW"])
def test_accumulation_spread_predicts_the_kernel_matrix_tolerances(mode, precision):
    """Teacher-forced logits of every job of tests/test_gpu_instantiations.py, summed in float32 and in float64 at the
    same operand precision: their largest difference estimates the accumulation-order noise a kernel may show, and the
    GPU tolerance must be at least 4 x that (fp16: at most the suite's 1e-3)."""
    model = helpers.make_model(0, mode)
    w = O.hot_weights(helpers.state_numpy(model))
    taps = model.upsample_taps(torch.device("cpu")).numpy()
    spread = 0.0
    for n, tables in K.all_jobs():
        job = K.make_job(n, mode, taps, tables)
        _, l32 = K.emulate(w, job, precision)
        _, l64 = K.emulate(w, job, precision, accumulate="f64")
        assert np.isfinite(l32).all() and np.abs(l64).max() > 0.1
        spread = max(spread, float(np.abs(l32 - l64).max()))
    tol = K.LOGIT_TOL[(precision, mode)]
    print(f"{precision} {mode}: predicted accumulation spread of the teacher-forced logits {spread:.3e}; GPU tolerance {tol:.1e}")
    assert spread <= tol / 4
    if precision == "fp16":
        assert tol <= 1e-3
