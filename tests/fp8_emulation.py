"""The fp8 (e4m3) arithmetic contract, restated on the CPU beside oracle/contract.py, whose folded order and
epilogues it reuses.  No engine serves it (DESIGN.md section 9): it exists to measure that precision's quality.

- All six K = H chains (CHAINS) take e4m3 operands.  The activations h1', h2', y1 and y2 are rounded by e4m3_round
  (RNE, saturating at +-448 like cvt.rn.satfinite.e4m3x2.f32).  Each weight row r is stored as e4m3(W_r / s_r), with
  s_r = max|W_r| / 448 computed in float64 and kept as float32 (1 for an all-zero row).
- Each column's float32 sum is multiplied by its s_r, then the bias and the epilogues follow as in fp16.
- The conditioning chain pre = Q cond + qk + x vq (K = 208) stays fp16."""
from __future__ import annotations

import numpy as np

from oracle import contract as C

F32 = np.float32
E4M3_MAX = 448.0
CHAINS = ("W2x", "W1h", "F1x", "W2h", "F2x", "F3")


def e4m3_round(x: np.ndarray) -> np.ndarray:
    """RNE float -> e4m3 (OCP FP8: 4 exponent bits, bias 7, 3 mantissa bits) -> float32, saturating to +-448.  Normal
    numbers (|x| >= 2^-6) are spaced 2^(e - 3) in the binade [2^e, 2^(e + 1)), subnormals 2^-9; the division by that
    power of two, the tie-to-even rint and the product are exact in float64."""
    x = np.clip(np.asarray(x, dtype=np.float64), -E4M3_MAX, E4M3_MAX)
    _, e = np.frexp(x)                                     # |x| = m 2^e, 0.5 <= m < 1: binade 2^(e - 1)
    q = np.ldexp(1.0, np.maximum(e - 4, -9))
    return (np.rint(x / q) * q).astype(F32)


def row_scales(W: np.ndarray) -> np.ndarray:
    """Per-row weight scales s_r = max|W_r| / 448 (float64, stored as float32); an all-zero row gets 1."""
    m = np.abs(np.asarray(W, dtype=np.float64)).max(axis=1)
    return np.where(m > 0, m / E4M3_MAX, 1.0).astype(F32)


def e4m3_rows(W: np.ndarray):
    """(e4m3(W_r / s_r) as float32, s) for every row r: the division in float64 by the stored float32 scale."""
    s = row_scales(W)
    return e4m3_round(np.asarray(W, dtype=np.float64) / s.astype(np.float64)[:, None]), s


def generate_segments(w: dict, mels_up, aux, *, n_seg, seg_len, seg_stride, uniforms=None, mode="MOL", expo=None,
                      x_force=None, want_logits=False, steps=None, fold_row0=None, fold_row_end=None, accumulate="f32"):
    """contract.generate_segments's signature and semantics (without `precision`), fp8 arithmetic."""
    f = C.fold_weights(w)
    H, G3 = C.H, 3 * C.H
    q16 = C.fp16_round(f["Q"].astype(F32))
    mats, scale = {}, {}
    for k in CHAINS:
        mats[k], scale[k] = e4m3_rows(f[k].astype(F32))
    if accumulate == "f64":
        mats_t = {k: np.ascontiguousarray(v.T, dtype=np.float64) for k, v in mats.items()}
        mm = lambda a, k: (a.astype(np.float64) @ mats_t[k]).astype(F32) * scale[k]
        mq = lambda a: (a.astype(np.float64) @ q16.T.astype(np.float64)).astype(F32)
    else:
        assert accumulate == "f32", accumulate
        mm = lambda a, k: (a @ mats[k].T).astype(F32) * scale[k]
        mq = lambda a: (a @ q16.T).astype(F32)
    B, S = n_seg, (steps if steps is not None else seg_len)
    L = mels_up.shape[0]
    n_classes = f["F3"].shape[0]
    cond_z = np.concatenate([np.concatenate([mels_up, aux], axis=1).astype(F32), np.zeros((1, C.CDIM), F32)])
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
        cond = C.fp16_round(cond_z[np.where(row < end, row, L)])
        if x_force is not None and t > 0:
            x = x_force[t - 1].reshape(B, 1).astype(F32)
        pre = (mq(cond) + f["qk"] + x * f["vq"]).astype(F32)
        h1 = C._gru(pre[:, :G3], gh1, h1)
        h1o = e4m3_round(h1)
        gi2 = mm(h1o, "W2x") + pre[:, G3:2 * G3]
        gh1 = mm(h1o, "W1h") + f["b1h"]
        fc1p = mm(h1o, "F1x")
        h2 = C._gru(gi2, gh2, h2)
        h2o = e4m3_round(h2)
        y1 = np.maximum(fc1p + mm(h2o, "F1x") + pre[:, 2 * G3:2 * G3 + H], 0).astype(F32)
        gh2 = mm(h2o, "W2h") + f["b2h"]
        y2 = np.maximum(mm(e4m3_round(y1), "F2x") + pre[:, 2 * G3 + H:], 0).astype(F32)
        logits = (mm(e4m3_round(y2), "F3") + f["b3"]).astype(F32)
        if want_logits:
            logits_all[t] = logits
        if mode == "MOL":
            u = uniforms[t]
            s = C.mol_sample(logits, u[:10 * B].reshape(B, 10), u[10 * B:11 * B])
        else:
            s, _ = C.raw_sample(logits, expo[t], n_classes)
        out[:, t] = s
        x = s.reshape(B, 1)
    return (out, logits_all) if want_logits else out


def emulate_job(w, job, accumulate="f32"):
    """kernel_jobs.emulate at fp8: (samples (n, STEPS), logits (STEPS, n, classes))."""
    import kernel_jobs as K
    return generate_segments(w, job["m_up"], job["aux"], n_seg=job["n"], seg_len=K.SEG_LEN, seg_stride=K.STRIDE,
                             steps=K.STEPS, mode=job["mode"], uniforms=job["uniforms"], expo=job["expo"],
                             x_force=job["x_force"], fold_row0=job["fold_row0"], fold_row_end=job["fold_row_end"],
                             want_logits=True, accumulate=accumulate)
