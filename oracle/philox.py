"""Host restatement of the engines' in-kernel draws (numpy): Philox4x32-10 and the word -> float maps of
wavernn_b200/csrc/wrnn_device.cuh, keyed exactly as wrnn_tc.cu, wrnn_stream.cu and wrnn_simt.cu key them.

Keying (every engine): counter = (step t, global fold seg_first + f, block, offset), key = (seed & 0xffffffff, seed >> 32).
- MoL: blocks 0, 1, 2; their words x, y, z, w, x, y, ... are mixture draws 0..9 and then the logistic draw.
- RAW: class c reads word c % 4 of block 16 + c // 4 and turns it into an Exp(1) draw -log(u01_open(word)).

Every float is produced exactly as the device produces it, so the arrays returned here can be handed to the engines'
explicit-draw paths (`uniforms`, `expo`) and must reproduce a Philox-mode run bit for bit."""
from __future__ import annotations

import numpy as np

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
MASK = np.uint64(0xFFFFFFFF)
RAW_BLOCK0 = 16                      # first Philox block of the RAW head's draws

F32 = np.float32
U_LO = F32(1e-5)                     # the reference's uniform_(1e-5, 1 - 1e-5) (utils/distribution.py:106, 118)
U_SPAN = F32(1.0) - F32(2e-5)        # (1.0f - 2e-5f) as the device folds it
U01_MAX_OPEN = F32(1.0) - F32(2.0 ** -24)   # largest float32 below 1


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Vectorised Philox4x32-10 (Salmon et al. 2011; the round and key schedule of wrnn_device.cuh).  Arguments are
    broadcastable integer arrays or scalars holding 32-bit values; returns four uint32 arrays (x, y, z, w)."""
    c0, c1, c2, c3, k0, k1 = np.broadcast_arrays(*[np.asarray(v, dtype=np.uint64) & MASK for v in (c0, c1, c2, c3, k0, k1)])
    c0, c1, c2, c3, k0, k1 = (a.copy() for a in (c0, c1, c2, c3, k0, k1))
    for _ in range(10):
        p0 = M0 * c0                     # < 2^64: exact in uint64
        p1 = M1 * c2
        n0 = (p1 >> np.uint64(32)) ^ c1 ^ k0
        n2 = (p0 >> np.uint64(32)) ^ c3 ^ k1
        c0, c1, c2, c3 = n0, p1 & MASK, n2, p0 & MASK
        k0 = (k0 + W0) & MASK
        k1 = (k1 + W1) & MASK
    return tuple(a.astype(np.uint32) for a in (c0, c1, c2, c3))


def u01(words):
    """((float)(x >> 8) + 0.5f) * 2^-24 in float32.  The float32 sum rounds to nearest even above 2^23, so the
    top word 0xffffffxx maps to exactly 1.0; the smallest value is 2^-25."""
    m = (np.asarray(words, dtype=np.uint32) >> np.uint32(8)).astype(F32)
    return ((m + F32(0.5)) * F32(2.0 ** -24)).astype(F32)


def u01_open(words):
    """u01 clamped below 1 (the RAW head's Exp(1) draws): the open interval (0, 1), so -log u > 0 for every word."""
    return np.minimum(u01(words), U01_MAX_OPEN)


def u_ref_range(words):
    """u01(x) * (1 - 2e-5f) + 1e-5f as the device computes it: one fused multiply-add.  The exact product and sum fit
    in 50 bits, so evaluating in float64 and rounding once to float32 equals the FFMA bit for bit."""
    return (u01(words).astype(np.float64) * np.float64(U_SPAN) + np.float64(U_LO)).astype(F32)


def _key(seed):
    seed = int(seed)
    return seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF


def mol_words(seed, offset, seg_first, n_seg, steps):
    """(S, B, 12) uint32: the words of blocks 0, 1, 2 for every (step, fold) (the 12th word is unused)."""
    k0, k1 = _key(seed)
    t = np.arange(steps, dtype=np.uint64)[:, None, None]
    g = (np.uint64(seg_first) + np.arange(n_seg, dtype=np.uint64))[None, :, None]
    blk = np.arange(3, dtype=np.uint64)[None, None, :]
    x, y, z, w = philox4x32_10(t, g, blk, int(offset) & 0xFFFFFFFF, k0, k1)
    return np.stack([x, y, z, w], axis=-1).reshape(steps, n_seg, 12)


def mol_uniforms(seed, offset, seg_first, n_seg, steps):
    """float32 (S, 11*B) in the `uniforms` layout (row t = [B x 10 mixture | B logistic], as helpers.replay_uniforms
    and the engines' explicit-draw path): the draws a Philox-mode MoL run makes."""
    u = u_ref_range(mol_words(seed, offset, seg_first, n_seg, steps))
    return np.concatenate([u[:, :, :10].reshape(steps, 10 * n_seg), u[:, :, 10]], axis=1)


def raw_words(seed, offset, seg_first, n_seg, steps, n_classes=512):
    """(S, B, n_classes) uint32: class c is word c % 4 of block 16 + c // 4."""
    k0, k1 = _key(seed)
    t = np.arange(steps, dtype=np.uint64)[:, None, None]
    g = (np.uint64(seg_first) + np.arange(n_seg, dtype=np.uint64))[None, :, None]
    blk = np.uint64(RAW_BLOCK0) + np.arange(n_classes // 4, dtype=np.uint64)[None, None, :]
    x, y, z, w = philox4x32_10(t, g, blk, int(offset) & 0xFFFFFFFF, k0, k1)
    return np.stack([x, y, z, w], axis=-1).reshape(steps, n_seg, n_classes)


def raw_expo(seed, offset, seg_first, n_seg, steps, n_classes=512):
    """(S, B, n_classes) float32 Exp(1) draws -logf(u01_open(word)) of a Philox-mode RAW run, and the words.  The
    device's logf is correctly rounded to within 1 ulp, so these match its draws to about 1 ulp (not bit for bit)."""
    words = raw_words(seed, offset, seg_first, n_seg, steps, n_classes)
    return (-np.log(u01_open(words).astype(np.float64))).astype(F32), words


def zero_draw_events(seed, offset, seg_first, n_seg, steps, n_classes=512, chunk=256):
    """(fold, step, class) of every RAW word whose u01 is exactly 1.0 (x >> 8 == 0xffffff), in (fold, step) order:
    the draws that were -0.0 before the Exp(1) draws were clamped into the open interval."""
    ev = []
    for t0 in range(0, steps, chunk):
        s = min(chunk, steps - t0)
        k0, k1 = _key(seed)
        t = (np.uint64(t0) + np.arange(s, dtype=np.uint64))[:, None, None]
        g = (np.uint64(seg_first) + np.arange(n_seg, dtype=np.uint64))[None, :, None]
        blk = np.uint64(RAW_BLOCK0) + np.arange(n_classes // 4, dtype=np.uint64)[None, None, :]
        words = np.stack(philox4x32_10(t, g, blk, int(offset) & 0xFFFFFFFF, k0, k1), axis=-1).reshape(s, n_seg, n_classes)
        for ts, f, c in zip(*np.nonzero((words >> np.uint32(8)) == np.uint32(0xFFFFFF))):
            ev.append((int(f), int(t0 + ts), int(c)))
    return sorted(ev)
