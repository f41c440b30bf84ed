"""The fp8 (e4m3) contract of tests/fp8_emulation.py, on the CPU: its rounder against torch.float8_e4m3fn, its per-row weight
scales against a float64 restatement, the accumulation spread that would set an fp8 kernel's tolerance, a negative
control of that tolerance, and what e4m3 chains do to the shipped checkpoint's likelihood of its own samples.  That
last measurement is why no engine serves fp8 (DESIGN.md section 9)."""
import numpy as np
import pytest
import torch

import fp8_emulation as E
import helpers
import kernel_jobs as K
from oracle import contract as C
from oracle import wavernn_oracle as O

# Teacher-forced logits of an fp8 kernel against fp8_emulation.generate_segments on the kernel_jobs jobs:
# at least 4 x the largest float32-vs-float64 accumulation spread of the emulation on those jobs
# (test_fp8_accumulation_spread_and_the_negative_control prints it: 7.4e-3 MoL / 1.26e-2 RAW).  No kernel serves
# fp8 (DESIGN §9): this is the bound one would be held to.
LOGIT_TOL_FP8 = {"MOL": 3.2e-2, "RAW": 5.6e-2}


def e4m3_codes():
    """Every finite e4m3 value, as float32, ascending (the 0x7f / 0xff codes are NaN)."""
    b = torch.arange(256, dtype=torch.int32).to(torch.uint8)
    v = b.view(torch.float8_e4m3fn).to(torch.float32).numpy()
    return np.unique(v[np.isfinite(v)])


def torch_e4m3(x):
    x = np.clip(np.asarray(x, np.float32), -E.E4M3_MAX, E.E4M3_MAX)
    return torch.from_numpy(x).to(torch.float8_e4m3fn).to(torch.float32).numpy()


def test_e4m3_rounder_equals_torch_on_every_code_every_midpoint_and_past_the_range():
    codes = e4m3_codes()
    assert codes.size == 253 and codes.max() == 448 and codes.min() == -448        # +-0 collapse to one value
    assert np.array_equal(E.e4m3_round(codes), codes)
    pos = codes[codes >= 0]                                  # pos[i] is the value of code i
    mid = ((pos[:-1].astype(np.float64) + pos[1:]) / 2).astype(np.float32)          # exact in float32
    got = E.e4m3_round(np.concatenate([mid, -mid]))
    assert np.array_equal(got, torch_e4m3(np.concatenate([mid, -mid])))
    # ties to even: the midpoint of codes i and i + 1 goes to the even one of the two
    i = np.arange(mid.size)
    assert np.array_equal(got[:mid.size], np.where(i % 2 == 0, pos[:-1], pos[1:]))
    assert np.array_equal(got[mid.size:], -got[:mid.size])
    rs = np.random.RandomState(8)
    beyond = np.concatenate([[448.0, 463.99, 464.0, 480.0, 1e4, 3e38, np.inf], rs.uniform(448, 1e6, 1000)]).astype(np.float32)
    beyond = np.concatenate([beyond, -beyond])
    assert np.array_equal(np.abs(E.e4m3_round(beyond)), np.full(beyond.size, 448, np.float32))
    assert np.array_equal(E.e4m3_round(beyond), torch_e4m3(beyond))
    sub = np.concatenate([rs.uniform(-2.0 ** -6, 2.0 ** -6, 20000), 2.0 ** -np.arange(6, 14), [2.0 ** -10, 3 * 2.0 ** -11]]).astype(np.float32)
    assert np.array_equal(E.e4m3_round(sub), torch_e4m3(sub))
    assert E.e4m3_round(np.float32(2.0 ** -10)) == 0 and E.e4m3_round(np.float32(3 * 2.0 ** -11)) == 2.0 ** -9
    wide = (rs.standard_normal(200000) * np.exp(rs.uniform(-12, 7, 200000))).astype(np.float32)
    assert np.array_equal(E.e4m3_round(wide), torch_e4m3(wide))


def test_row_scales_restate_max_abs_over_448_and_the_rows_use_the_stored_scale():
    rs = np.random.RandomState(3)
    W = (rs.standard_normal((64, 512)) * 1e-2).astype(np.float32)
    W[5] = 0
    W[6, :] = 0; W[6, 17] = -3e-3                                                    # the max is negative
    W[7] *= 1e4                                                                      # beyond e4m3 unscaled
    q, s = E.e4m3_rows(W)
    for r in range(W.shape[0]):
        m = max(abs(float(v)) for v in W[r])
        want = np.float32(m / 448.0) if m > 0 else np.float32(1.0)
        assert s[r] == want and s.dtype == np.float32
        qr = np.array([float(E.e4m3_round(np.float64(v) / np.float64(s[r]))) for v in W[r]])
        assert np.array_equal(q[r], qr.astype(np.float32))
    assert np.abs(q).max() == 448 and not q[5].any() and s[5] == 1
    # the scaled rows keep the weights out of e4m3's subnormal range, which unscaled rounding of 1e-2 weights is in
    rel = np.abs(q * s[:, None] - W)[8:] / np.abs(W[8:]).max(axis=1, keepdims=True)
    assert rel.max() <= 2.0 ** -4 * 1.0001
    small = (np.abs(W) < 2.0 ** -7) & (np.arange(64) >= 8)[:, None]
    rel_elem = lambda a: np.median(np.abs(a - W)[small] / np.abs(W[small]))
    assert rel_elem(E.e4m3_round(W)) > 4 * rel_elem(q * s[:, None])


@pytest.mark.parametrize("mode", ["MOL", "RAW"])
def test_fp8_accumulation_spread_and_the_negative_control(mode):
    """Teacher-forced logits of every job of the kernel matrix (tests/kernel_jobs.py) at fp8, summed in float32 and in
    float64: an fp8 kernel's tolerance against the emulation must be at least 4 x their largest difference.

    Negative control: the fp8 emulation is far outside the fp16 tolerance of the fp16 one.  The converse does not hold
    for a max-error bound: the fp16 emulation is only about 2.5 x the fp8 spread from the fp8 one, inside LOGIT_TOL_FP8,
    because e4m3 rounding flips of the activations under another sum order move a logit by as much as the fp8-vs-fp16
    difference (as bf16 against fp16, tests/test_contract.py).  The mean logit error separates them: the float64-summed
    emulation, standing in for a kernel with another sum order, is at least 4 x closer to the fp8 emulation on average
    than to the fp16 one."""
    model = helpers.make_model(0, mode)
    w = O.hot_weights(helpers.state_numpy(model))
    taps = model.upsample_taps(torch.device("cpu")).numpy()
    spread = shift = 0.0
    own, other = [], []
    for n, tables in K.all_jobs():
        job = K.make_job(n, mode, taps, tables)
        _, l32 = E.emulate_job(w, job)
        _, l64 = E.emulate_job(w, job, accumulate="f64")
        _, l16 = K.emulate(w, job, "fp16")
        assert np.isfinite(l32).all() and np.abs(l64).max() > 0.1
        spread = max(spread, float(np.abs(l32 - l64.astype(np.float64)).max()))
        shift = max(shift, float(np.abs(l32 - l16.astype(np.float64)).max()))
        own.append(np.abs(l64 - l32.astype(np.float64)).ravel()); other.append(np.abs(l64 - l16.astype(np.float64)).ravel())
    own, other = float(np.concatenate(own).mean()), float(np.concatenate(other).mean())
    print(f"fp8 {mode}: accumulation spread {spread:.3e} (tolerance {LOGIT_TOL_FP8[mode]:.1e}); fp8 vs fp16 emulation "
          f"{shift:.3e} (fp16 tolerance {K.LOGIT_TOL[('fp16', mode)]:.1e}); mean error of the float64-summed stand-in "
          f"against the fp8 / fp16 emulation {own:.2e} / {other:.2e}")
    assert spread <= LOGIT_TOL_FP8[mode] / 4
    assert shift > 10 * K.LOGIT_TOL[("fp16", mode)]
    assert own <= other / K.ROUNDING_SEPARATION


# ---------------------------------------------------------------------------------------------------------------------
# quality on the shipped checkpoint: teacher-forced on the reference's own free-running samples
# ---------------------------------------------------------------------------------------------------------------------
MOL_BINS = 65536          # the MoL head is trained on 16-bit targets: a sample's bin is 2 / (MOL_BINS - 1) wide


def _log_sigmoid(a):
    return -np.logaddexp(0.0, -a)


def mol_nll(logits, x, log_scale_min=O.LOG_SCALE_MIN):
    """Negative log-likelihood (nats) of samples x in [-1, 1] under the discretized mixture of logistics of each row of
    logits (..., 30) = [10 mixture logits | 10 means | 10 log scales], in float64.  Component k puts mass
    sigmoid((x + d - mu_k) / s_k) - sigmoid((x - d - mu_k) / s_k) on x's bin, d = 1 / (MOL_BINS - 1); the lowest bin
    (x < -0.999) takes the whole lower tail and the highest (x > 0.999) the upper one.  Log scales are clamped below at
    log(1e-14) as the sampler clamps them."""
    lg = np.asarray(logits, np.float64)
    pi, mu = lg[..., :10], lg[..., 10:20]
    ls = np.maximum(lg[..., 20:30], log_scale_min)
    x = np.asarray(x, np.float64)[..., None]
    d = 1.0 / (MOL_BINS - 1)
    inv = np.exp(-ls)
    hi, lo = inv * (x - mu + d), inv * (x - mu - d)
    # log(sigmoid(hi) - sigmoid(lo)) = log sigmoid(hi) + log(1 - exp(log sigmoid(lo) - log sigmoid(hi))), and the same
    # with the mirrored arguments where both lie in the upper tail (no cancellation in either)
    up = lo > 0
    a, b = np.where(up, -lo, hi), np.where(up, -hi, lo)
    with np.errstate(divide="ignore"):
        mid = _log_sigmoid(a) + np.log(-np.expm1(_log_sigmoid(b) - _log_sigmoid(a)))
    # where the bin is narrow against the scale, the difference underflows: density at x times the bin's width
    c = inv * (x - mu)
    dens = c - ls - 2 * np.logaddexp(0.0, c) + np.log(2 * d)
    mid = np.where(np.isfinite(mid), mid, dens)
    lp = np.where(x < -0.999, _log_sigmoid(hi), np.where(x > 0.999, _log_sigmoid(-lo), mid))
    log_pi = pi - np.logaddexp.reduce(pi, axis=-1, keepdims=True)
    return -np.logaddexp.reduce(log_pi + lp, axis=-1)


def test_mol_nll_restates_the_discretized_logistic():
    """mol_nll against a direct sum of bin masses (float64, no tails or cancellation guards), on rows where the
    direct form is exact enough, and the whole distribution sums to one over the bins."""
    rs = np.random.RandomState(0)
    lg = np.concatenate([rs.randn(3, 10), rs.uniform(-0.5, 0.5, (3, 10)), rs.uniform(-6, -2, (3, 10))], 1)
    edges = np.linspace(-1, 1, MOL_BINS)
    d = 1.0 / (MOL_BINS - 1)
    sig = lambda a: 1 / (1 + np.exp(-a))
    for r in range(3):
        pi = np.exp(lg[r, :10] - np.logaddexp.reduce(lg[r, :10]))
        mu, s = lg[r, 10:20], np.exp(lg[r, 20:30])
        hi = sig((edges[:, None] + d - mu) / s); lo = sig((edges[:, None] - d - mu) / s)
        hi[-1], lo[0] = 1.0, 0.0
        mass = (pi * (hi - lo)).sum(1)
        assert abs(mass.sum() - 1) < 1e-9
        pick = np.arange(0, MOL_BINS, 997)
        pick = pick[mass[pick] > 1e-9]                      # where the direct difference of sigmoids keeps its digits
        got = mol_nll(np.repeat(lg[r:r + 1], pick.size, 0), edges[pick])
        np.testing.assert_allclose(got, -np.log(mass[pick]), rtol=1e-6, atol=0)


@pytest.fixture(scope="module")
def trained_teacher_forced():
    """Teacher-forced logits (12,100, 4, 30) of the shipped checkpoint at each precision, on the Tacotron fixture mel,
    fed the reference's own free-running samples of that mel (the `raw` array of trained_tacotron.npz)."""
    model = helpers.make_model(0, "MOL", "cpu")
    missing = model.load_state_dict(helpers.pretrained_state_dict(), strict=False)
    assert not missing.missing_keys and not missing.unexpected_keys
    sd = helpers.state_numpy(model)
    w = O.hot_weights(sd)
    g = helpers.load_golden("trained_tacotron.npz")
    mel = helpers.tacotron_mels()[int(g["sentence"])]
    m_up, aux = O.upsample_network(sd, O.pad_time(mel.T, 2).T, pad=2)
    U = helpers.replay_uniforms(int(g["seed"]), 12100, 4)
    raw = g["raw"]
    out = {}
    kw = dict(n_seg=4, seg_len=12100, seg_stride=11550, uniforms=U, x_force=raw.T.copy(), want_logits=True)
    for p in ("fp32", "fp16", "bf16"):
        _, out[p] = C.generate_segments(w, m_up, aux, precision=p, **kw)
    _, out["fp8"] = E.generate_segments(w, m_up, aux, **kw)
    return out, raw


def test_fp8_degrades_the_shipped_checkpoints_likelihood_of_its_own_samples(trained_teacher_forced):
    """What fp8 chains do to audio quality, before any kernel is written: the mean per-sample NLL of the reference's
    samples under each precision's logits, and the |logit| change against fp32.

    Measured (DESIGN §5): median NLL fp32 4.747, fp16 4.774, bf16 4.787, fp8 5.561 nats; mean 10.32 / 9.23 / 8.34 / 24.45
    (the mean is carried by a few samples that land far out in a narrow component, so it moves either way under any
    rounding; fp8 moves it up by 14 nats); samples whose NLL moves by more than 1 nat from fp32: 4.6 % / 5.1 % / 37.7 %;
    median |logit change| 1.9e-4 / 1.5e-3 / 2.7e-2.  fp16 and bf16 leave the likelihood where fp32 has it; fp8 is clearly
    worse than bf16, so no engine serves it.  The pins below hold these conclusions with a margin."""
    lgs, raw = trained_teacher_forced
    nll = {p: mol_nll(lg, raw.T) for p, lg in lgs.items()}
    med = {p: float(np.median(v)) for p, v in nll.items()}
    moved, dmed = {}, {}
    for p in ("fp16", "bf16", "fp8"):
        e = np.abs(lgs[p].astype(np.float64) - lgs["fp32"])
        moved[p] = float((np.abs(nll[p] - nll["fp32"]) > 1).mean())
        dmed[p] = float(np.median(e))
        print(f"{p}: |logit - fp32 logit| max {e.max():.3e} p99.9 {np.quantile(e, 0.999):.3e} median {dmed[p]:.3e}; "
              f"NLL nats / sample mean {nll[p].mean():.4f} median {med[p]:.4f} (fp32 {nll['fp32'].mean():.4f} / "
              f"{med['fp32']:.4f}); samples moved by > 1 nat {moved[p]:.4f}")
    for p in ("fp16", "bf16"):
        assert abs(med[p] - med["fp32"]) <= 0.1 and moved[p] <= 0.1
    assert dmed["fp16"] <= 1e-3 and dmed["bf16"] <= 5e-3 and dmed["fp8"] >= 1e-2
    assert med["fp8"] >= med["bf16"] + 0.5 and moved["fp8"] >= 0.25
    assert nll["fp8"].mean() >= 2 * nll["bf16"].mean()
