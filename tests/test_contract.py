"""The engine-arithmetic emulation (folded order, fp16/bf16 operand rounding) against the
reference-order oracle.  States the FP tolerance of the product path on the CPU."""
import hashlib

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


@pytest.mark.parametrize("precision", ["fp16", "bf16", "fp32"])
@pytest.mark.parametrize("mode", ["MOL", "RAW"])
def test_accumulation_spread_predicts_the_kernel_matrix_tolerances(mode, precision):
    """Teacher-forced logits of every job of tests/test_gpu_instantiations.py and tests/test_gpu_simt.py, summed in
    float32 and in float64 at the same operand precision: their largest difference estimates the accumulation-order
    noise a kernel may show, and the GPU tolerance must be at least 4 x that (fp16: at most the suite's 1e-3)."""
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


@pytest.mark.parametrize("mode", ["MOL", "RAW"])
def test_reference_order_spread_predicts_the_strict_engine_bound(mode):
    """The fp32 emulation (folded order, float32 and float64 sums) against wavernn_oracle.generate_segments (the
    reference's unfolded order) on every job of the kernel matrix: the SIMT engine's fp32 bound against that order,
    kernel_jobs.ORACLE_TOL, must be at least 4 x their largest difference.  The oracle has no fold tables, so it reads
    each job's windows re-laid out by kernel_jobs.oracle_rows; the emulation on those rows equals the emulation on the
    job bit for bit (the re-layout reads exactly the job's rows)."""
    model = helpers.make_model(0, mode)
    w = O.hot_weights(helpers.state_numpy(model))
    taps = model.upsample_taps(torch.device("cpu")).numpy()
    spread = 0.0
    for n, tables in K.all_jobs():
        job = K.make_job(n, mode, taps, tables)
        _, l32 = K.emulate(w, job, "fp32")
        _, l64 = K.emulate(w, job, "fp32", accumulate="f64")
        _, lo = K.emulate_oracle(w, job)
        m, a = K.oracle_rows(job)
        _, lr = C.generate_segments(w, m, a, n_seg=n, seg_len=K.STEPS, seg_stride=K.STEPS, steps=K.STEPS, mode=mode,
                                    uniforms=job["uniforms"], expo=job["expo"], x_force=job["x_force"], want_logits=True,
                                    precision="fp32")
        assert np.array_equal(lr, l32), (n, tables)
        spread = max(spread, float(np.abs(l32 - lo.astype(np.float64)).max()), float(np.abs(l64 - lo.astype(np.float64)).max()))
    tol = K.ORACLE_TOL[mode]
    print(f"fp32 {mode}: emulation vs the reference order {spread:.3e}; GPU bound {tol:.1e}")
    assert spread <= tol / 4


@pytest.mark.parametrize("mode", ["MOL", "RAW"])
def test_operand_rounding_of_another_precision_fails_the_kernel_matrix_checks(mode):
    """Negative control of the SIMT matrix (tests/test_gpu_simt.py): a handle that rounded its operands to another
    type than its own must fail the comparison with its own emulation.

    fp32: the fp16 and bf16 emulations differ from the fp32 one by more than 10 x the fp32 tolerance, so the strict
    engine's max-error check catches either rounding.

    fp16 / bf16: the bf16 emulation differs from the fp16 one by only ~2.5 x the fp16 tolerance (1.5e-3 MoL, 1.7e-3 RAW
    on these small random-init logits), and by less than the bf16 tolerance.  Most of the bf16 accumulation spread is
    an activation whose bf16 rounding flips when the sum order changes, so a bf16 max-error bound cannot be tighter than
    the bf16-vs-fp16 shift.  The 16-bit handles are therefore also checked on the MEAN logit error: against the
    emulation at their own precision it must be at most a quarter of that against the other 16-bit precision.  The
    float64-summed emulation stands in for a kernel with another sum order here; it must pass that check by 10 x."""
    model = helpers.make_model(0, mode)
    w = O.hot_weights(helpers.state_numpy(model))
    taps = model.upsample_taps(torch.device("cpu")).numpy()
    shift = {("fp16", "fp32"): 0.0, ("bf16", "fp32"): 0.0, ("bf16", "fp16"): 0.0}
    mean = {(p, q): [] for p in ("fp16", "bf16") for q in ("fp16", "bf16")}        # (stand-in precision, emulation)
    for n, tables in K.all_jobs():
        job = K.make_job(n, mode, taps, tables)
        l = {p: K.emulate(w, job, p)[1].astype(np.float64) for p in ("fp32", "fp16", "bf16")}
        for a, b in shift:
            shift[(a, b)] = max(shift[(a, b)], float(np.abs(l[a] - l[b]).max()))
        for p in ("fp16", "bf16"):
            _, l64 = K.emulate(w, job, p, accumulate="f64")
            for q in ("fp16", "bf16"):
                mean[(p, q)].append(np.abs(l64 - l[q]).ravel())
    mean = {k: float(np.concatenate(v).mean()) for k, v in mean.items()}
    print(f"{mode}: max logit shift fp16 vs fp32 {shift[('fp16', 'fp32')]:.3e}, bf16 vs fp32 {shift[('bf16', 'fp32')]:.3e} "
          f"(10 x fp32 tolerance {10 * K.LOGIT_TOL[('fp32', mode)]:.1e}); bf16 vs fp16 {shift[('bf16', 'fp16')]:.3e} "
          f"(fp16 tolerance {K.LOGIT_TOL[('fp16', mode)]:.1e}); mean error of the float64-summed stand-in against its own / "
          f"the other 16-bit emulation: fp16 {mean[('fp16', 'fp16')]:.2e} / {mean[('fp16', 'bf16')]:.2e}, "
          f"bf16 {mean[('bf16', 'bf16')]:.2e} / {mean[('bf16', 'fp16')]:.2e}")
    assert shift[("fp16", "fp32")] > 10 * K.LOGIT_TOL[("fp32", mode)]
    assert shift[("bf16", "fp32")] > 10 * K.LOGIT_TOL[("fp32", mode)]
    assert shift[("bf16", "fp16")] > 2 * K.LOGIT_TOL[("fp16", mode)]
    for p, q in (("fp16", "bf16"), ("bf16", "fp16")):
        assert mean[(p, p)] <= mean[(p, q)] / 10, (p, mean)
    assert K.ROUNDING_SEPARATION <= 4


# ---------------------------------------------------------------------------------------------------------------------
# the kernel matrix's jobs at upsampling geometries other than (5, 5, 11)
# ---------------------------------------------------------------------------------------------------------------------
# sha256 (first 16 hex digits) of every hop-275 job as kernel_jobs made it before it took a hop, on fixed taps
HOP_275_JOBS = {
    (24, False, "MOL"): "40284be60d698699", (24, True, "MOL"): "7b6044de4f34e70f", (25, False, "MOL"): "505c9cd82b995bd1",
    (25, True, "MOL"): "813469b9decfc47d", (73, False, "MOL"): "673e009efd4e8a23", (73, True, "MOL"): "eaa21d3279c97b0e",
    (17, False, "MOL"): "85e557183166e59d", (17, True, "MOL"): "ad48a914fe80806f", (33, False, "MOL"): "a419ac708f3dfe86",
    (33, True, "MOL"): "c660abc597a4baf5", (24, False, "RAW"): "0428ae144e970448", (24, True, "RAW"): "584be791aeffad2d",
    (25, False, "RAW"): "b4b71983da14b850", (25, True, "RAW"): "40c3e97ef1aa4ad3", (73, False, "RAW"): "fe0a79ad2934b78e",
    (73, True, "RAW"): "3658f95c8a9ebb88", (17, False, "RAW"): "531433ebe116c2f5", (17, True, "RAW"): "60e7f0412296b061",
    (33, False, "RAW"): "6cc976dfd0bc9ab1", (33, True, "RAW"): "c72f6f6e4ef28d67",
}


def _job_digest(job):
    h = hashlib.sha256()
    for k in sorted(job):
        v = job[k]
        if isinstance(v, np.ndarray):
            h.update(k.encode()); h.update(str(v.dtype).encode()); h.update(str(v.shape).encode())
            h.update(np.ascontiguousarray(v).tobytes())
        elif k != "hop":
            h.update(f"{k}={v!r}".encode())
    return h.hexdigest()[:16]


def test_hop_275_jobs_are_unchanged():
    """Every job of the hop-275 kernel matrix, bit for bit, by default and with hop=275 spelled out (fixed taps, so that
    the digests do not depend on torch's CPU convolutions)."""
    taps = np.random.RandomState(275).rand(275, 5).astype(np.float32)
    for mode in ("MOL", "RAW"):
        for n, tables in K.all_jobs():
            job = K.make_job(n, mode, taps, tables)
            assert job["hop"] == K.HOP and _job_digest(job) == HOP_275_JOBS[(n, tables, mode)], (n, tables, mode)
            assert _job_digest(K.make_job(n, mode, taps, tables, hop=K.HOP)) == HOP_275_JOBS[(n, tables, mode)]


@pytest.mark.parametrize("hop", sorted(K.GEOMETRIES))
def test_jobs_at_other_hops_have_the_edges(hop):
    """The jobs at another hop keep the edges of the 275 ones: fold windows that start at many phases, windows of the
    tables that end mid-frame, frames that cover the stream's last row (mel frames up to T + 3)."""
    for n, tables in K.all_jobs():
        job = K.make_job(n, "MOL", K.geometry_taps(hop), tables, hop=hop)
        L, T = job["L"], job["T"]
        assert job["hop"] == hop and job["mel_frames"].shape == (T + 4, 80) and (L - 1) // hop + 4 <= T + 3
        row0 = job["fold_row0"] if tables else (K.SEG_FIRST + np.arange(n)) * K.STRIDE
        assert len(set((row0 % hop).tolist())) >= min(hop, n) // (2 if tables else 1), "fold windows start at few phases"
        if tables and hop > 1:
            assert (job["fold_row_end"] % hop != 0).all()
        rows = job["m_up"].shape[0]
        assert rows == L - job["row_lo"] and job["aux"].shape == (rows, 128)


def _spread(w, job, precision):
    _, l32 = K.emulate(w, job, precision)
    _, l64 = K.emulate(w, job, precision, accumulate="f64")
    assert np.isfinite(l32).all() and np.abs(l64).max() > 0.1
    return float(np.abs(l32 - l64).max())


@pytest.mark.parametrize("precision", ["fp16", "bf16"])
@pytest.mark.parametrize("mode", ["MOL", "RAW"])
@pytest.mark.parametrize("hop", K.KERNEL_HOPS)
def test_accumulation_spread_predicts_the_tolerances_at_other_hops(hop, mode, precision):
    """test_accumulation_spread_predicts_the_kernel_matrix_tolerances on the jobs of tests/test_gpu_geometries.py: the
    same model and LOGIT_TOL, rows formed at another hop with that geometry's taps."""
    w = O.hot_weights(helpers.state_numpy(helpers.make_model(0, mode)))
    taps = K.geometry_taps(hop)
    spread = max(_spread(w, K.make_job(n, mode, taps, tables, hop=hop), precision) for n, tables in K.all_jobs())
    tol = K.LOGIT_TOL[(precision, mode)]
    print(f"hop {hop} {precision} {mode}: predicted accumulation spread of the teacher-forced logits {spread:.3e}; "
          f"GPU tolerance {tol:.1e}")
    assert spread <= tol / 4


@pytest.mark.parametrize("mode", ["MOL", "RAW"])
@pytest.mark.parametrize("hop", K.KERNEL_HOPS)
def test_rows_formed_at_the_wrong_hop_move_the_logits_past_the_tolerance(hop, mode):
    """Negative control of the GPU comparison at another hop: the emulation on the rows a kernel would form with the
    hop-275 table, or at the right hop one phase late, moves the teacher-forced logits by more than 10 x LOGIT_TOL
    (the larger, bf16 one), so a kernel that used a stale hop or phase would fail the comparison."""
    w = O.hot_weights(helpers.state_numpy(helpers.make_model(0, mode)))
    taps, taps_275 = K.geometry_taps(hop), K.geometry_taps(K.HOP)
    bound = 10 * max(K.LOGIT_TOL[(p, mode)] for p in ("fp16", "bf16"))
    shifts = {"hop 275": 0.0, "phase + 1": 0.0}
    for n, tables in ((24, False), (25, True)):
        job = K.make_job(n, mode, taps, tables, hop=hop)
        _, want = K.emulate(w, job, "fp16")
        lo, n_rows = job["row_lo"], job["L"] - job["row_lo"]
        T_275 = job["L"] // K.HOP + 1
        mel = np.zeros((max(T_275, job["T"]) + 4, 80), np.float32)
        aux = np.zeros((max(T_275, job["T"]) + 4, 128), np.float32)
        mel[:job["T"] + 4], aux[:job["T"] + 4] = job["mel_frames"], job["aux_frames"]
        wrong = {"hop 275": C.expand_rows(mel, aux, taps_275, K.HOP, lo, n_rows),
                 "phase + 1": C.expand_rows(job["mel_frames"], job["aux_frames"], taps, hop, lo + 1, n_rows)}
        for what, (m, a) in wrong.items():
            _, lg = K.emulate(w, dict(job, m_up=m.astype(np.float32), aux=a.astype(np.float32)), "fp16")
            shifts[what] = max(shifts[what], float(np.abs(lg.astype(np.float64) - want).max()))
    print(f"hop {hop} {mode}: logit shift on rows formed at hop 275 {shifts['hop 275']:.3e}, one phase late "
          f"{shifts['phase + 1']:.3e}; 10 x tolerance {bound:.1e}")
    assert shifts["hop 275"] > bound and shifts["phase + 1"] > bound
