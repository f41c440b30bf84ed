"""The reference's training loss per sample (train_wavernn.py:83) restated in numpy float32, in the reference's order:
what wrnn_score computes on the device, checked against the reference itself by tests/golden/score_pins.npz."""
from __future__ import annotations

import numpy as np

from oracle.wavernn_oracle import LOG_SCALE_MIN

F32 = np.float32


def _softplus(x):
    """F.softplus (beta 1, threshold 20)."""
    with np.errstate(over="ignore"):
        return np.where(x > F32(20), x, np.log1p(np.exp(x, dtype=F32), dtype=F32)).astype(F32)


def mol_loss(logits: np.ndarray, y: np.ndarray, num_classes: int = 65536) -> np.ndarray:
    """utils/distribution.py:16-84, discretized_mix_logistic_loss(y_hat, y, reduce=False): the per-sample loss in nats
    of targets y (B,) under the mixtures logits (B, 30) = [10 mixture logits | 10 means | 10 log-scales], with
    log_scale_min = log(1e-14).  Every branch of the reference: y < -0.999 (log_cdf_plus), y > 0.999
    (log_one_minus_cdf_min), cdf_delta > 1e-5 (log(clamp(cdf_delta, 1e-12))), else log_pdf_mid - log(32767.5).  The
    reference blends them with 0/1 masks; each is finite, so the blend is the selection.  Python scalars enter torch's
    float32 arithmetic rounded to float32, as here."""
    lg = np.asarray(logits, dtype=F32)
    y = np.asarray(y, dtype=F32)[:, None]
    nr = lg.shape[1] // 3
    logit_probs, means = lg[:, :nr], lg[:, nr:2 * nr]
    log_scales = np.maximum(lg[:, 2 * nr:3 * nr], F32(LOG_SCALE_MIN))                      # :32
    centered_y = y - means                                                                 # :37
    inv_stdv = np.exp(-log_scales, dtype=F32)                                              # :38
    half_bin = F32(1. / (num_classes - 1))
    plus_in = inv_stdv * (centered_y + half_bin)                                           # :39
    cdf_plus = (F32(1) / (F32(1) + np.exp(-plus_in, dtype=F32))).astype(F32)
    min_in = inv_stdv * (centered_y - half_bin)                                            # :41
    with np.errstate(over="ignore"):
        cdf_min = (F32(1) / (F32(1) + np.exp(-min_in, dtype=F32))).astype(F32)
    log_cdf_plus = plus_in - _softplus(plus_in)                                            # :46
    log_one_minus_cdf_min = -_softplus(min_in)                                             # :50
    cdf_delta = cdf_plus - cdf_min                                                         # :53
    mid_in = inv_stdv * centered_y                                                         # :55
    log_pdf_mid = mid_in - log_scales - F32(2) * _softplus(mid_in)                         # :58
    inner_inner = np.where(cdf_delta > F32(1e-5), np.log(np.maximum(cdf_delta, F32(1e-12)), dtype=F32),
                           log_pdf_mid - F32(np.log((num_classes - 1) / 2)))               # :74-76
    inner = np.where(y > F32(0.999), log_one_minus_cdf_min, inner_inner)                   # :77-78
    log_probs = np.where(y < F32(-0.999), log_cdf_plus, inner)                             # :79-80
    mx = logit_probs.max(axis=1, keepdims=True)                                            # F.log_softmax
    log_softmax = (logit_probs - mx) - np.log(np.exp(logit_probs - mx, dtype=F32).sum(axis=1, keepdims=True, dtype=F32), dtype=F32)
    log_probs = log_probs + log_softmax                                                    # :82
    m = log_probs.max(axis=1)                                                              # log_sum_exp, :6-12
    lse = m + np.log(np.exp(log_probs - m[:, None], dtype=F32).sum(axis=1, dtype=F32), dtype=F32)
    return (-lse).astype(F32)                                                              # :87


def raw_label(y: np.ndarray, n_classes: int) -> np.ndarray:
    """The class of a target sample (the inverse of label_2_float, utils/dataset.py:88):
    rint((y + 1) (n_classes - 1) / 2), clamped to [0, n_classes - 1]."""
    v = np.rint((np.asarray(y, dtype=F32) + F32(1)) * F32(n_classes - 1) * F32(0.5))
    return np.clip(v, 0, n_classes - 1).astype(np.int64)


def raw_loss(logits: np.ndarray, y: np.ndarray) -> np.ndarray:
    """F.cross_entropy(logits, label, reduction='none') (train_wavernn.py:83, RAW head): -log_softmax(logits)[label],
    label = raw_label(y).  logits (B, n_classes), y (B,)."""
    lg = np.asarray(logits, dtype=F32)
    k = raw_label(y, lg.shape[1])
    mx = lg.max(axis=1)
    s = np.exp(lg - mx[:, None], dtype=F32).sum(axis=1, dtype=F32)
    return (-((lg[np.arange(lg.shape[0]), k] - mx) - np.log(s, dtype=F32))).astype(F32)


ULPS = 32   # expf / logf / log1pf each round within 1-2 ulp on the device and in numpy; several roundings reach a term


def mol_loss_tolerance(logits: np.ndarray, y: np.ndarray, num_classes: int = 65536):
    """Per-sample bound on |kernel - mol_loss| for the same logits: ULPS units of 2^-24 of the largest intermediate term
    of the evaluation -- the log-probabilities, the mixture logits, the argument of the branch taken and, in the
    cdf_delta branch, (1 + |plus_in|) max(cdf_plus, cdf_min) / cdf_delta: an ulp of plus_in or min_in moves a cdf by
    that argument's magnitude in its own ulps, which cdf_delta's cancellation magnifies by max(cdf) / cdf_delta.
    A component whose cdf_delta lies so close to 1e-5 that two evaluations may take different branches adds the
    difference of the two branch values (the bin's approximation error, not a rounding); the mask of such samples is
    returned too."""
    lg = np.asarray(logits, dtype=np.float64)
    y64 = np.asarray(y, dtype=np.float64)[:, None]
    nr = lg.shape[1] // 3
    ls = np.maximum(lg[:, 2 * nr:], LOG_SCALE_MIN)
    inv = np.exp(-ls)
    c = y64 - lg[:, nr:2 * nr]
    hb = 1.0 / (num_classes - 1)
    plus_in, min_in, mid_in = inv * (c + hb), inv * (c - hb), inv * c
    with np.errstate(over="ignore"):
        cp, cm = 1 / (1 + np.exp(-plus_in)), 1 / (1 + np.exp(-min_in))
    delta = cp - cm
    with np.errstate(divide="ignore", invalid="ignore"):
        main = np.where(delta > 0, np.maximum(cp, cm) / np.where(delta > 0, delta, 1), 0.0)
    main = main * (1 + np.maximum(np.abs(plus_in), np.abs(min_in)))
    sp = np.where(mid_in > 20, mid_in, np.log1p(np.exp(np.minimum(mid_in, 20))))
    pdf = np.abs(mid_in) + np.abs(ls) + 2 * sp + 11
    # a component at the 1e-5 branch may take either branch: both branches' terms and the two values' difference enter
    # the bound
    delta_err = ULPS * 2.0 ** -24 * (1 + np.maximum(np.abs(plus_in), np.abs(min_in))) * np.maximum(cp, cm)
    near = (np.abs(delta - 1e-5) <= delta_err) & (np.abs(y64) <= 0.999)
    inner = np.where(near, np.maximum(main + 12, pdf), np.where(delta > 1e-5, main + 12, pdf))
    term = np.where(y64 < -0.999, np.abs(plus_in), np.where(y64 > 0.999, np.abs(min_in), inner))
    scale = np.maximum.reduce([np.ones(len(lg)), np.abs(lg[:, :nr]).max(1), term.max(1),
                               np.abs(mol_loss(logits, y)).astype(np.float64) + 1])
    with np.errstate(divide="ignore", invalid="ignore"):
        jump = np.abs(np.log(np.maximum(delta, 1e-12)) - (mid_in - ls - 2 * sp - np.log((num_classes - 1) / 2)))
    extra = np.where(near, np.nan_to_num(jump, nan=0.0, posinf=0.0), 0.0).max(1)
    return ULPS * 2.0 ** -24 * scale + extra, near.any(1)


def raw_loss_tolerance(logits: np.ndarray) -> np.ndarray:
    """Per-sample bound on |kernel - raw_loss| for the same logits: ULPS units of 2^-24 of the largest of |logit| and
    log(n_classes) (the terms of max + log(sum) - logit)."""
    lg = np.asarray(logits, dtype=np.float64)
    return ULPS * 2.0 ** -24 * np.maximum(np.abs(lg).max(1), np.log(lg.shape[1]) + 1)


def mol_sensitivity(logits: np.ndarray) -> np.ndarray:
    """1 + the largest inverse scale exp(-max(log_scale, log(1e-14))) among a sample's components: how far the loss of
    a sample moves per unit of error in its logits (a mean off by e moves that component's cdf arguments by e / scale).
    Two fp32 evaluations of the same network differ in the logits' last bits, so on trained weights, whose log-scales
    reach the clamp, their losses can differ by hundreds of nats; measured against the reference the bound is a
    multiple of this."""
    ls = np.maximum(np.asarray(logits, dtype=np.float64)[:, 20:30], LOG_SCALE_MIN)
    return 1.0 + np.exp(-ls).max(1)
