"""The Griffin-Lim edge tests' mels, error measure and wrong restatements, on the grid of tests/mel_edges.py (every
configuration wrnn_mel_create accepts, at its ends and at odd interior values).  Shared by tests/test_gl_edges.py (the
oracle and the kernels' code run on the host) and tests/test_gpu_gl_edges.py (the kernels).

Everything is deterministic; the restatements take the arguments of gl_oracle.reconstruct_waveform."""
from __future__ import annotations

import functools

import numpy as np
import scipy.fft
import scipy.signal

import gl_oracle as G
import helpers
import mel_oracle as MO
from mel_edges import GRID, cfg  # noqa: F401  (the grid is mel_edges'; re-exported for the Griffin-Lim tests)
from oracle import philox

F32, F64 = np.float32, np.float64
TINY = np.finfo(F32).tiny
SEED = 7
# The largest local_steps allowed between two implementations of the same path, per n_iter.
# n_iter 0: the output is linear in S.  The kernels and the oracle share S, the phases, the complex64 products and the
# float32 window sum-square w bit for bit (float64 window squares added in frame order); their float64 inverse
# transforms differ below 2^-40 of a frame's peak.  So the undivided sums Y differ only where one float32 addition
# rounds the other way, 1 step of a partial sum, and a partial sum is of the size of the largest undivided magnitude
# over the frames that cover the sample.  The division by w rounds once on each side, half a step of y each, at most 1
# step of Y after multiplying back by w.  2 steps in all; 4 leaves room for a partial sum above the scale.  Measured on
# the grid: 1.0 (sr8k-fft256-mels128, where S differs in its last bit, host run and device alike), 0.2 on the device
# at sr16k-fmin7990, 0 elsewhere.
# n_iter 1 and 2: the analysis of a signal that differs by those steps moves each rebuilt bin by a few float32 steps of
# its frame's spectrum, and the phase of a weak bin moves by that over its own magnitude; the second phase update
# compounds the first.  Measured on the grid, host run and device alike: 2.5 and 14.7 (both at fft256-mels128).
# 8 and 64 leave a factor of 3 and 4.
LOCAL_TOL = {0: 4, 1: 8, 2: 64}


def shortest(c):
    """The fewest frames wrnn_griffinlim_many accepts: hop_length * (T - 1) > n_fft / 2."""
    return (c["n_fft"] // 2) // c["hop_length"] + 2


def speech(n):
    """The speech fixture's first n samples (tiled where it is shorter)."""
    x = helpers.load_golden("trained_tacotron.npz")["wav"].astype(F32)
    return np.tile(x, n // x.size + 1)[:n] if n > x.size else x[:n]


def out_of_range(mel):
    """mel with every third value (every value of a mel of fewer than 12) replaced, in turn, by -1, -inf, 2 and +inf."""
    m = np.array(mel, F32)
    flat = m.reshape(-1)
    idx = np.arange(0, flat.size, 3 if flat.size >= 12 else 1)
    flat[idx] = np.array([-1, -np.inf, 2, np.inf], F32)[np.arange(idx.size) % 4]
    return m


def mels(c):
    """The mels of configuration c (all keys): name -> float32 [n_mels, T].  The oracle's analysis of the speech fixture
    at about 40 frames (not at hop_length 1, where that is shorter than the shortest T) and cut to the shortest T; a
    silent and a full-scale mel, and an out-of-range one, at the shortest T."""
    hop, N = c["hop_length"], c["n_fft"]
    T0 = shortest(c)
    out = {}
    if hop > 1:
        out["speech"] = MO.melspectrogram(speech(max(40 * hop, N)), **c)
    short = MO.melspectrogram(speech(hop * (T0 - 1)), **c)
    assert short.shape[1] == T0
    out["shortest"] = short
    out["silent"] = np.zeros_like(short)
    out["full"] = np.ones_like(short)
    out["out_of_range"] = out_of_range(short)
    return out


# ---- the error measure ------------------------------------------------------------------------------------------------
def _range_max(a, lo, hi):
    """max(a[lo[i] .. hi[i]]) for each i (inclusive, lo <= hi), by a sparse table."""
    levels = [a]
    while 2 ** len(levels) <= a.size:
        p, s = levels[-1], 2 ** (len(levels) - 1)
        levels.append(np.maximum(p[:-s], p[s:]))
    k = np.floor(np.log2(hi - lo + 1)).astype(int)
    out = np.empty(lo.size, F64)
    for j in np.unique(k):
        sel = k == j
        out[sel] = np.maximum(levels[j][lo[sel]], levels[j][hi[sel] - 2 ** j + 1])
    return out


def local_steps(got, ref, c):
    """Per output sample: |got - ref| times the oracle's float32 window sum-square w (undoing the division, so the
    difference is in the units the frames are added in), in float32 steps of the largest undivided magnitude |ref| w
    over the frames that cover the sample.  Samples where w <= float32 tiny are left undivided by both sides and must
    match exactly: 0 if they do, inf if not.  Two NaNs match; one NaN is inf."""
    got, ref = np.asarray(got, F32), np.asarray(ref, F32)
    N, hop = c["n_fft"], c["hop_length"]
    L = ref.size
    T = L // hop + 1
    assert got.shape == ref.shape and L == hop * (T - 1)
    w = G.window_sumsquare(T, **c)[N // 2:N // 2 + L].astype(F64)
    U = np.zeros(N + hop * (T - 1))                      # the undivided magnitudes in padded coordinates
    with np.errstate(invalid="ignore"):
        U[N // 2:N // 2 + L] = np.nan_to_num(np.abs(ref.astype(F64)) * w, nan=0.0, posinf=np.finfo(F64).max)
    p = np.arange(L) + N // 2
    i0 = np.maximum(0, -((N - 1 - p) // hop))           # ceil((p - N + 1) / hop)
    i1 = np.minimum(T - 1, p // hop)
    covered = i0 <= i1
    scale = np.zeros(L)
    scale[covered] = _range_max(U, i0[covered] * hop, i1[covered] * hop + N - 1)
    same = (got == ref) | (np.isnan(got) & np.isnan(ref))
    with np.errstate(invalid="ignore", over="ignore"):
        d = np.abs(got.astype(F64) - ref.astype(F64)) * w / np.spacing(scale.astype(F32)).astype(F64)
    d = np.where(same, 0.0, np.where(np.isnan(d), np.inf, d))
    exact = w <= TINY
    return np.where(exact, np.where(same, 0.0, np.inf), d)


def peak_steps(got, ref):
    """The former measure: max |got - ref| in float32 steps of the output's peak."""
    return float(np.abs(got - ref).max() / np.spacing(np.abs(ref).max()))


@functools.lru_cache(maxsize=8)
def phases(seed, T, n_bins):
    """gl_oracle.phases, kept: the Philox draws dominate the oracle's time at hop_length 1.  Read only."""
    ph = G.phases(seed, T, n_bins)
    ph.flags.writeable = False
    return ph


_S_CACHE = {}


def magnitudes(mel, **c):
    """gl_oracle.mel_to_stft (the FISTA solve), kept per mel and configuration: the solve dominates the oracle's time
    at hop_length 1.  Read only."""
    mel = np.ascontiguousarray(mel, F32)
    key = (mel.shape, mel.tobytes(), tuple(sorted(dict(MO.DEFAULT, **c).items())))
    if key not in _S_CACHE:
        if len(_S_CACHE) >= 16:
            _S_CACHE.clear()
        _S_CACHE[key] = G.mel_to_stft(mel, **c)
        _S_CACHE[key].flags.writeable = False
    return _S_CACHE[key]


def oracle(mel, n_iter, seed=SEED, **c):
    """gl_oracle.reconstruct_waveform (the FISTA solve), step for step."""
    c = dict(MO.DEFAULT, **c)
    S = magnitudes(mel, **c)
    return G.griffinlim(S, phases(seed, S.shape[1], S.shape[0]), n_iter, **c)


# ---- wrong restatements ---------------------------------------------------------------------------------------------
def _solve(A, B, *, pivot_drop=G.PIVOT_DROP, iters=G.FISTA_ITERS, gershgorin=False):
    """gl_oracle.nnls_fista with its constants as arguments."""
    A64, B64 = np.asarray(A, F64), np.asarray(B, F64)
    Gm = A64 @ A64.T
    M = Gm.shape[0]
    inv_d, sub, prev_d = np.zeros(M), np.zeros(M), 0.0
    for m in range(M):
        l = Gm[m, m - 1] / prev_d if m > 0 and prev_d > 0 else 0.0
        d = Gm[m, m] - l * Gm[m, m - 1] if m > 0 else Gm[m, m]
        if not d > pivot_drop * Gm[m, m]:
            l, d = 0.0, 0.0
        sub[m], inv_d[m], prev_d = l, (1.0 / d if d > 0 else 0.0), d
    if gershgorin:
        off = np.abs(np.diag(Gm, 1))
        step = 1.0 / (np.diag(Gm) + np.r_[0.0, off] + np.r_[off, 0.0]).max()
    else:
        step = 1.0 / np.linalg.eigvalsh(Gm)[-1]
    u = np.empty_like(B64)
    for m in range(M):
        u[m] = B64[m] - (sub[m] * u[m - 1] if m else 0.0)
    z = u * inv_d[:, None]
    for m in range(M - 2, -1, -1):
        z[m] -= sub[m + 1] * z[m + 1]
    x = np.maximum(A64.T @ z, 0.0)
    y, t = x.copy(), 1.0
    for _ in range(iters):
        xn = np.maximum(y - (A64.T @ (A64 @ y - B64)) * step, 0.0)
        tn = (1.0 + np.sqrt(1.0 + 4.0 * t * t)) / 2.0
        y = xn + ((t - 1.0) / tn) * (xn - x)
        x, t = xn, tn
    return x.astype(F32)


def _phases_bin_frame(seed, T, n_bins):
    """gl_oracle.phases with the Philox counter's first two words swapped: keyed by (bin, frame)."""
    k0, k1 = int(seed) & 0xFFFFFFFF, (int(seed) >> 32) & 0xFFFFFFFF
    t = np.arange(T, dtype=np.uint64)[None, :]
    blk = (np.arange(n_bins, dtype=np.uint64) // np.uint64(4))[:, None]
    words = np.stack(philox.philox4x32_10(blk, t, 0, 0, k0, k1), axis=0)
    w = np.take_along_axis(words, (np.arange(n_bins) % 4)[None, :, None].repeat(T, axis=2), axis=0)[0]
    return np.exp(2j * np.pi * philox.u01(w).astype(F64)).astype(np.complex64)


def _symmetric_window(n_fft, win_length, **_):
    w = scipy.signal.get_window("hann", win_length, fftbins=False)
    lp = (n_fft - win_length) // 2
    return np.pad(w, (lp, n_fft - win_length - lp))


def _irfft_keeping_dc_nyquist_imag(X, n):
    """The kernels' packed inverse (an n / 2-point transform of the (even, odd) sample pairs) without dropping the
    imaginary parts of bins 0 and n / 2; with them dropped it is irfft."""
    H = n // 2
    k = np.arange(H)[:, None]
    pk, pm = X[:H], X[H - np.arange(H)]
    er, ei = 0.5 * (pk.real + pm.real), 0.5 * (pk.imag - pm.imag)
    dr, di = 0.5 * (pk.real - pm.real), 0.5 * (pk.imag + pm.imag)
    wr, wi = np.cos(-2 * np.pi * k / n), np.sin(-2 * np.pi * k / n)
    orr, oi = dr * wr + di * wi, di * wr - dr * wi
    R = scipy.fft.fft((er - oi) - 1j * (ei + orr), axis=0)
    y = np.empty((n,) + X.shape[1:])
    y[0::2], y[1::2] = R.real / H, -R.imag / H
    return y


def _restated(mel, n_iter=32, seed=0, *, phases=phases, window=None, tiny=True, irfft=None, trim=0,
              momentum=G.MOMENTUM / (1 + G.MOMENTUM), eps=1e-16, clip=True, pivot_drop=G.PIVOT_DROP,
              iters=G.FISTA_ITERS, gershgorin=False, pad="reflect", ola=F32, wss=F32, stages=False, **cfg):
    """reconstruct_waveform with one step done wrong; the defaults restate gl_oracle.reconstruct_waveform bit for bit.
    stages: return the outputs after 0, 1, ..., n_iter iterations instead (one pass)."""
    c = dict(MO.DEFAULT, **cfg)
    N, hop, W = c["n_fft"], c["hop_length"], c["win_length"]
    mel = np.asarray(mel, F32)
    L = F32(c["min_level_db"])
    d = (np.clip(mel, F32(0), F32(1)) if clip else mel) * -L + L
    if clip and (pivot_drop, iters, gershgorin) == (G.PIVOT_DROP, G.FISTA_ITERS, False):
        S = magnitudes(mel, **c)
    else:
        with np.errstate(over="ignore", invalid="ignore"):
            B = np.power(10.0, (d * F32(0.05)).astype(F64)).astype(F32)
            S = _solve(G.fb32(**c), B, pivot_drop=pivot_drop, iters=iters, gershgorin=gershgorin)
    T = S.shape[1]
    win_a = MO.window(N, W)
    win_s = win_a if window is None else window(N, W)
    wsum = np.zeros(N + hop * (T - 1), dtype=wss)
    for i in range(T):
        wsum[i * hop:i * hop + N] += win_s ** 2

    def istft(X):
        Xc = X.astype(np.complex128)
        frames = (scipy.fft.irfft(Xc, n=N, axis=0) if irfft is None else irfft(Xc, N)) * win_s[:, None]
        y = np.zeros(N + hop * (T - 1), dtype=ola)
        for i in range(T):
            y[i * hop:i * hop + N] += frames[:, i]
        nz = wsum > TINY if tiny else np.ones(wsum.size, bool)
        with np.errstate(invalid="ignore", divide="ignore"):
            y[nz] /= wsum[nz]
        return y[N // 2 + trim:N // 2 + trim + hop * (T - 1)].astype(F32)

    def stft(y):
        yp = np.pad(y, N // 2, mode=pad)
        fr = yp[np.arange(N)[:, None] + hop * np.arange(T)[None]].astype(F64)
        return scipy.fft.rfft(win_a[:, None] * fr, axis=0).astype(np.complex64)

    angles = phases(seed, T, S.shape[0])
    rebuilt, outs = 0.0, []
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        for _ in range(n_iter):
            tprev = rebuilt
            outs.append(istft(S * angles))
            rebuilt = stft(outs[-1])
            angles = (rebuilt - momentum * tprev).astype(np.complex64)
            angles /= np.abs(angles) + F32(eps) if eps else np.abs(angles)
        outs.append(istft(S * angles))
    return outs if stages else outs[-1]


# the visible slips: each must miss LOCAL_TOL in at least one cell of the grid.  A float64 overlap-add or sum-square
# shows where many frames overlap: at hop_length 1, 2048 float32 additions per sample round far from one float64 sum.
WRONG = {
    "phases_keyed_bin_frame": lambda m, n, s, **c: _restated(m, n, s, phases=_phases_bin_frame, **c),
    "symmetric_window_in_istft": lambda m, n, s, **c: _restated(m, n, s, window=_symmetric_window, **c),
    "no_tiny_test": lambda m, n, s, **c: _restated(m, n, s, tiny=False, **c),
    "centre_trim_one_off": lambda m, n, s, **c: _restated(m, n, s, trim=1, **c),
    "momentum_0.99": lambda m, n, s, **c: _restated(m, n, s, momentum=G.MOMENTUM, **c),
    "no_1e-16": lambda m, n, s, **c: _restated(m, n, s, eps=0.0, **c),
    "denormalize_without_clip": lambda m, n, s, **c: _restated(m, n, s, clip=False, **c),
    "fista_99_steps": lambda m, n, s, **c: _restated(m, n, s, iters=G.FISTA_ITERS - 1, **c),
    "gershgorin_step": lambda m, n, s, **c: _restated(m, n, s, gershgorin=True, **c),
    "constant_padding_in_stft": lambda m, n, s, **c: _restated(m, n, s, pad="constant", **c),
    "float64_overlap_add": lambda m, n, s, **c: _restated(m, n, s, ola=F64, **c),
    "float64_sum_square": lambda m, n, s, **c: _restated(m, n, s, wss=F64, **c),
}
# slips the output cannot show, each for a reason of its own; they stay inside LOCAL_TOL everywhere.
# - the imaginary parts of the DC and Nyquist bins: a Slaney triangle is 0 at its edges and no band reaches below
#   fmin >= 0 or past the Nyquist frequency, so the float32 filterbank's weight in both bins is 0 (3e-18 at most, at
#   44,100 Hz) and so is S there;
# - the pivot drop: the pivots it drops on this grid (fft256-mels128, fft256-hop1, sr8k-fft256-mels128: bands that
#   repeat a neighbour's single bin) are 1e-20 to 1e-18 of their diagonals; kept, they change the start of the solve,
#   and 100 FISTA steps land on the same float32 S.
INVISIBLE = {
    "irfft_keeps_dc_nyquist_imag": lambda m, n, s, **c: _restated(m, n, s, irfft=_irfft_keeping_dc_nyquist_imag, **c),
    "no_pivot_drop": lambda m, n, s, **c: _restated(m, n, s, pivot_drop=0.0, **c),
}
