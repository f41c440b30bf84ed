"""Numpy emulation of the ENGINE'S arithmetic contract -- TEST INFRASTRUCTURE ONLY.

`wavernn_oracle.generate_segments` restates the reference in its own operation order
(fp32).  The CUDA engines compute the same function in the folded order of
wavernn_b200/csrc/wrnn_fold.h and, in fp16/bf16 mode, round every tensor-core operand to
that type.  This module restates THAT order on the CPU so the kernels can be checked far more
tightly (accumulation-order noise only) than against the fp32 reference order, and so the
size of the bf16 deviation can be measured on the CPU.  It is derived from the reference
lines cited in wrnn_fold.h; it is validated against `wavernn_oracle` (fp32 mode must
agree to ~1e-6) in tests/test_contract.py.
"""
from __future__ import annotations

import numpy as np

from .wavernn_oracle import F32, LOG_SCALE_MIN, mol_sample, raw_sample  # noqa: F401

H, FEAT, AUXD = 512, 80, 32
F1IN = FEAT + AUXD
CDIM = FEAT + 4 * AUXD


def bf16_round(x: np.ndarray) -> np.ndarray:
    """Round-to-nearest-even float32 -> bfloat16 -> float32."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    u = x.view(np.uint32).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000
    return u.astype(np.uint32).view(np.float32).reshape(x.shape)


def fp16_round(x: np.ndarray) -> np.ndarray:
    """RNE float32 -> IEEE half -> float32 (saturating to +-65504 like cvt.rn.satfinite)."""
    x = np.clip(np.asarray(x, dtype=np.float32), -65504.0, 65504.0)
    return x.astype(np.float16).astype(np.float32)


def rounder(precision: str):
    return {"fp16": fp16_round, "bf16": bf16_round, "fp32": lambda a: np.asarray(a, dtype=F32)}[precision]


def fold_weights(w: dict) -> dict:
    """Double-precision folding, same formulas as wrnn_fold.h::fold()."""
    d = {k: np.asarray(v, dtype=np.float64) for k, v in w.items()}
    I_w, bI = d["I.weight"], d["I.bias"]
    i0, Ic = I_w[:, 0], I_w[:, 1:]
    W1i, W1h = d["rnn1.weight_ih_l0"], d["rnn1.weight_hh_l0"]
    W2i, W2h = d["rnn2.weight_ih_l0"], d["rnn2.weight_hh_l0"]
    W2x, W2a = W2i[:, :H], W2i[:, H:]
    F1x, F1a = d["fc1.weight"][:, :H], d["fc1.weight"][:, H:]
    F2x, F2a = d["fc2.weight"][:, :H], d["fc2.weight"][:, H:]
    G3 = 3 * H
    # Q: all conditioning rows in one [G3 + G3 + H + H, CDIM] matrix
    Q = np.zeros((2 * G3 + 2 * H, CDIM))
    Q[:G3, :F1IN] = W1i @ Ic
    Q[G3:2 * G3, :F1IN] = W2x @ Ic
    Q[G3:2 * G3, F1IN:F1IN + AUXD] = W2a
    Q[2 * G3:2 * G3 + H, :F1IN] = F1x @ Ic
    Q[2 * G3:2 * G3 + H, F1IN + AUXD:F1IN + 2 * AUXD] = F1a
    Q[2 * G3 + H:, F1IN + 2 * AUXD:] = F2a
    qk = np.concatenate([W1i @ bI + d["rnn1.bias_ih_l0"], W2x @ bI + d["rnn2.bias_ih_l0"],
                         F1x @ bI + d["fc1.bias"], d["fc2.bias"]])
    vq = np.concatenate([W1i @ i0, W2x @ i0, F1x @ i0, np.zeros(H)])
    return dict(Q=Q, qk=qk.astype(F32), vq=vq.astype(F32), W2x=W2x, W1h=W1h, F1x=F1x, W2h=W2h, F2x=F2x,
                F3=d["fc3.weight"], b1h=d["rnn1.bias_hh_l0"].astype(F32), b2h=d["rnn2.bias_hh_l0"].astype(F32),
                b3=d["fc3.bias"].astype(F32))


def _sig(x):
    return (F32(1) / (F32(1) + np.exp(-x, dtype=F32))).astype(F32)


def _gru(gi, gh, h):
    r = _sig(gi[:, :H] + gh[:, :H])
    z = _sig(gi[:, H:2 * H] + gh[:, H:2 * H])
    n = np.tanh(gi[:, 2 * H:] + r * gh[:, 2 * H:]).astype(F32)
    return ((F32(1) - z) * n + z * h).astype(F32)


def expand_rows(mel_frames, aux_frames, taps, hop, row_lo, n_rows):
    """Rows [row_lo, row_lo + n_rows) of the per-sample conditioning stream from frame-rate tensors, in float64:
    m[n] = sum_d taps[n % hop, d] * mel_frames[n // hop + d] and aux[n] = aux_frames[n // hop] (UpsampleNetwork's
    stretch+conv cascade as a 5-tap table per output phase; `WaveRNN.upsample_taps`).  mel_frames is the padded
    (T + 4, 80) mel, so the last row of a (T * hop)-row stream reads frames up to T + 3."""
    n = np.arange(row_lo, row_lo + n_rows)
    fr, ph = n // hop, n % hop
    taps = np.asarray(taps, dtype=np.float64)
    mel = np.asarray(mel_frames, dtype=np.float64)
    m = sum(taps[ph, d][:, None] * mel[fr + d] for d in range(5))
    return m, np.asarray(aux_frames, dtype=np.float64)[fr]


def generate_segments(w: dict, mels_up, aux, *, n_seg, seg_len, seg_stride, uniforms=None, mode="MOL",
                      expo=None, x_force=None, want_logits=False, steps=None, precision="fp16",
                      fold_row0=None, fold_row_end=None, accumulate="f32"):
    """Same signature/semantics as wavernn_oracle.generate_segments, engine arithmetic.

    fold_row0 / fold_row_end: per-fold conditioning windows (the engines' fold tables): fold f reads row
    fold_row0[f] + t, and rows at or past fold_row_end[f] as zero.  Without them fold f starts at f * seg_stride and
    rows at or past len(mels_up) are zero.
    accumulate: "f32" sums every matmul in float32 like the tensor cores' accumulators; "f64" sums in float64 and
    rounds once.  Their difference estimates the accumulation-order noise at a given operand precision."""
    f = fold_weights(w)
    rnd = rounder(precision)
    mats = {k: rnd(f[k].astype(F32)) for k in ("Q", "W2x", "W1h", "F1x", "W2h", "F2x", "F3")}
    if accumulate == "f64":
        mats_t = {k: np.ascontiguousarray(v.T, dtype=np.float64) for k, v in mats.items()}
        mm = lambda a, k: (a.astype(np.float64) @ mats_t[k]).astype(F32)
    else:
        assert accumulate == "f32", accumulate
        mm = lambda a, k: (a @ mats[k].T).astype(F32)
    B, S = n_seg, (steps if steps is not None else seg_len)
    L = mels_up.shape[0]
    G3 = 3 * H
    n_classes = f["F3"].shape[0]
    cond_z = np.concatenate([np.concatenate([mels_up, aux], axis=1).astype(F32), np.zeros((1, CDIM), F32)])
    if fold_row0 is None:
        base, end = np.arange(B) * seg_stride, np.full(B, L)
    else:
        base, end = np.asarray(fold_row0, dtype=np.int64), np.asarray(fold_row_end, dtype=np.int64)
        assert base.shape == end.shape == (B,) and end.max() <= L
    h1 = np.zeros((B, H), F32); h2 = np.zeros((B, H), F32)
    gh1 = np.tile(f["b1h"], (B, 1)); gh2 = np.tile(f["b2h"], (B, 1))
    x = np.zeros((B, 1), F32)
    out = np.zeros((B, S), F32)
    logits_all = np.zeros((S, B, n_classes), F32) if want_logits else None
    for t in range(S):
        row = base + t
        cond = rnd(cond_z[np.where(row < end, row, L)])
        if x_force is not None and t > 0:
            x = x_force[t - 1].reshape(B, 1).astype(F32)
        pre = (mm(cond, "Q") + f["qk"] + x * f["vq"]).astype(F32)
        h1 = _gru(pre[:, :G3], gh1, h1)
        h1o = rnd(h1)
        gi2 = mm(h1o, "W2x") + pre[:, G3:2 * G3]
        gh1 = mm(h1o, "W1h") + f["b1h"]
        fc1p = mm(h1o, "F1x")
        h2 = _gru(gi2, gh2, h2)
        h2o = rnd(h2)
        y1 = np.maximum(fc1p + mm(h2o, "F1x") + pre[:, 2 * G3:2 * G3 + H], 0).astype(F32)
        gh2 = mm(h2o, "W2h") + f["b2h"]
        y2 = np.maximum(mm(rnd(y1), "F2x") + pre[:, 2 * G3 + H:], 0).astype(F32)
        logits = (mm(rnd(y2), "F3") + f["b3"]).astype(F32)
        if want_logits:
            logits_all[t] = logits
        if mode == "MOL":
            u = uniforms[t]
            s = mol_sample(logits, u[:10 * B].reshape(B, 10), u[10 * B:11 * B])
        else:
            s, _ = raw_sample(logits, expo[t], n_classes)
        out[:, t] = s
        x = s.reshape(B, 1)
    return (out, logits_all) if want_logits else out
