"""numpy/scipy restatement of the reference's reconstruct_waveform(mel, n_iter) (utils/dsp.py:105-116) through librosa
0.7: denormalize and db_to_amp in float32, mel_to_stft (a non-negative least-squares inversion of the float32 Slaney
filterbank) and griffinlim (momentum 0.99) with the dtypes librosa 0.7 uses -- float64 FFTs, complex64 bins and phases,
a float32 signal overlap-added in frame order and divided by the float32 window sum-square.

Two NNLS solvers:
- nnls_lbfgs: librosa 0.7's own, restated (least-squares start clipped at 0, then fmin_l_bfgs_b with m = 1025 over
  blocks of 63 columns).  The reference arm: its minimiser is not unique and scipy's line search picks one.
- nnls_fista: the library's (wrnn_gl.cu), a fixed number of accelerated projected-gradient steps from the clipped
  minimum-norm least-squares start, with step 1 / lambda_max(A A^T).

The initial phases are the library's Philox draws (oracle/philox.py), keyed by (seed, frame, bin)."""
from __future__ import annotations

import numpy as np
import scipy.fft
import scipy.optimize

import mel_oracle as MO
from oracle import philox

F32, F64 = np.float32, np.float64
MOMENTUM = 0.99
FISTA_ITERS = 100            # wrnn_gl.cu's NNLS_ITERS
PIVOT_DROP = 1e-10           # a band whose pivot falls below this share of its diagonal is left out of the start solve
MAX_MEM_BLOCK = 2 ** 8 * 2 ** 10


# ---- the magnitudes ---------------------------------------------------------------------------------------------------
def fb32(sample_rate, n_fft, n_mels, fmin, **_):
    """librosa 0.7 filters.mel(sr, n_fft, n_mels, fmin, dtype=float32): each triangle stored as float32, then scaled by
    the float64 Slaney norm and stored as float32 again."""
    fft = np.linspace(0, sample_rate / 2, 1 + n_fft // 2, endpoint=True)
    mel_f = MO.mel_to_hz(np.linspace(MO.hz_to_mel(fmin), MO.hz_to_mel(sample_rate / 2), n_mels + 2))
    fdiff, ramps = np.diff(mel_f), np.subtract.outer(mel_f, fft)
    w = np.zeros((n_mels, 1 + n_fft // 2), dtype=F32)
    for i in range(n_mels):
        w[i] = np.maximum(0, np.minimum(-ramps[i] / fdiff[i], ramps[i + 2] / fdiff[i + 1]))
    w *= (2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels]))[:, None]
    return w


def amplitudes(mel, min_level_db=-100.0, **_):
    """db_to_amp(denormalize(mel)) as numpy 1.22 evaluates it on a float32 mel: float32 throughout."""
    mel = np.asarray(mel, dtype=F32)
    L = F32(min_level_db)
    d = (np.clip(mel, F32(0), F32(1)) * -L) + L
    # np.power(10.0, float32) is powf; the library rounds the float64 power, which is what a correctly rounded powf gives
    return np.power(10.0, (d * F32(0.05)).astype(F64)).astype(F32)


def nnls_lbfgs(A, B, dtype=F32):
    """librosa 0.7 util.nnls(A, B) for a matrix B: float32 [n_bins, T] (dtype=float64: each block's solution before
    librosa rounds it to float32)."""
    A, B = np.asarray(A, F32), np.asarray(B, F32)

    def obj(x, shape, A, B):
        diff = np.dot(A, x.reshape(shape)) - B
        return 0.5 * np.sum(diff ** 2), np.dot(A.T, diff).flatten()

    def block(B, x_init):
        x, _, _ = scipy.optimize.fmin_l_bfgs_b(obj, x_init, args=(x_init.shape, A, B), bounds=[(0, None)] * x_init.size,
                                               m=A.shape[1])
        return x.reshape(x_init.shape)

    n_columns = int(MAX_MEM_BLOCK // (A.shape[-1] * A.itemsize))
    if B.shape[-1] <= n_columns:
        x0 = np.clip(np.linalg.lstsq(A, B, rcond=None)[0], 0, None)
        return block(B, x0).astype(dtype)
    x_init = np.clip(np.linalg.lstsq(A, B, rcond=None)[0].astype(F32), 0, None)
    x = x_init.astype(dtype)
    for s in range(0, x.shape[-1], n_columns):
        t = min(s + n_columns, B.shape[-1])
        x[:, s:t] = block(B[:, s:t], x_init[:, s:t])
    return x


def solve_tables(A):
    """The constants of the library's solve, from the float32 filterbank A [n_mels, n_bins] in float64: the LDL^T factor
    of the tridiagonal A A^T (inverse pivots and subdiagonal multipliers; a dropped band has inverse pivot 0 and
    decouples its neighbours) and 1 / lambda_max(A A^T)."""
    A = np.asarray(A, F64)
    G = A @ A.T
    M = G.shape[0]
    inv_d, sub = np.zeros(M), np.zeros(M)
    prev_d = 0.0
    for m in range(M):
        l = G[m, m - 1] / prev_d if m > 0 and prev_d > 0 else 0.0
        d = G[m, m] - l * G[m, m - 1] if m > 0 else G[m, m]
        if not d > PIVOT_DROP * G[m, m]:
            l, d = 0.0, 0.0
        sub[m], inv_d[m], prev_d = l, (1.0 / d if d > 0 else 0.0), d
    lam = np.linalg.eigvalsh(G)[-1]
    return inv_d, sub, 1.0 / lam


def nnls_fista(A, B, iters=FISTA_ITERS, dtype=F32):
    """The library's NNLS, vectorised over frames: float32 A [n_mels, n_bins], float32 B [n_mels, T] -> float32
    [n_bins, T] (dtype=float64: the solution before the library rounds it)."""
    A64, B64 = np.asarray(A, F64), np.asarray(B, F64)
    inv_d, sub, step = solve_tables(A)
    M = A.shape[0]
    u = np.empty_like(B64)
    for m in range(M):                                       # L u = b
        u[m] = B64[m] - (sub[m] * u[m - 1] if m else 0.0)
    z = u * inv_d[:, None]                                   # D v = u
    for m in range(M - 2, -1, -1):                           # L^T z = v
        z[m] -= sub[m + 1] * z[m + 1]
    x = np.maximum(A64.T @ z, 0.0)
    y, t = x.copy(), 1.0
    for _ in range(iters):
        g = A64.T @ (A64 @ y - B64)
        xn = np.maximum(y - g * step, 0.0)
        tn = (1.0 + np.sqrt(1.0 + 4.0 * t * t)) / 2.0
        y = xn + ((t - 1.0) / tn) * (xn - x)
        x, t = xn, tn
    return x.astype(dtype)


def rel_residual(A, B, X):
    """Per frame 1/2 |A x - b|^2 / 1/2 |b|^2, in float64."""
    A, B, X = (np.asarray(v, F64) for v in (A, B, X))
    return ((A @ X - B) ** 2).sum(axis=0) / (B ** 2).sum(axis=0)


def mel_to_stft(mel, solver="fista", **cfg):
    """mel_to_stft(db_to_amp(denormalize(mel)), power=1): float32 [n_fft / 2 + 1, T]."""
    c = dict(MO.DEFAULT, **cfg)
    A, B = fb32(**c), amplitudes(mel, **c)
    return nnls_fista(A, B) if solver == "fista" else nnls_lbfgs(A, B)


# ---- the transforms ---------------------------------------------------------------------------------------------------
def window_sumsquare(T, *, n_fft, hop_length, win_length, dtype=F32, **_):
    """librosa 0.7 filters.window_sumsquare(..., dtype=float32): the float64 squared window added into float32, frame
    after frame."""
    w2 = MO.window(n_fft, win_length) ** 2
    x = np.zeros(n_fft + hop_length * (T - 1), dtype=dtype)
    for i in range(T):
        s = i * hop_length
        x[s:s + n_fft] += w2
    return x


def istft(X, *, n_fft, hop_length, win_length, dtype=F32, **_):
    """librosa 0.7 istft(X, center=True, dtype=float32): float64 irfft times the window, overlap-added into float32 in
    frame order, divided by the window sum-square where it exceeds float32 tiny, centre-trimmed: float32
    [hop_length * (T - 1)] (dtype=float64: the same in float64 throughout)."""
    T = X.shape[1]
    ytmp = MO.window(n_fft, win_length)[:, None] * scipy.fft.irfft(X.astype(np.complex128), n=n_fft, axis=0)
    y = np.zeros(n_fft + hop_length * (T - 1), dtype=dtype)
    for i in range(T):
        s = i * hop_length
        y[s:s + n_fft] += ytmp[:, i]
    wss = window_sumsquare(T, n_fft=n_fft, hop_length=hop_length, win_length=win_length, dtype=dtype)
    nz = wss > np.finfo(dtype).tiny
    y[nz] /= wss[nz]
    return y[n_fft // 2:-(n_fft // 2)]


def stft(y, *, n_fft, hop_length, win_length, dtype=F32, **_):
    """librosa 0.7 stft(y, center=True, pad_mode='reflect', dtype=complex64): [n_fft / 2 + 1, 1 + len(y) // hop]
    (dtype=float64: complex128 bins of a float64 signal)."""
    yp = np.pad(np.asarray(y, dtype), n_fft // 2, mode="reflect")
    T = 1 + (len(yp) - n_fft) // hop_length
    frames = yp[np.arange(n_fft)[:, None] + hop_length * np.arange(T)[None]].astype(F64)
    return scipy.fft.rfft(MO.window(n_fft, win_length)[:, None] * frames, axis=0).astype(np.result_type(dtype, 1j))


def phases(seed, T, n_bins):
    """The library's initial phases exp(2 pi i u) (complex64) [n_bins, T]: u is u01 of word k % 4 of the Philox block at
    counter (frame t, k // 4, 0, 0) under key seed."""
    k0, k1 = int(seed) & 0xFFFFFFFF, (int(seed) >> 32) & 0xFFFFFFFF
    t = np.arange(T, dtype=np.uint64)[None, :]
    blk = (np.arange(n_bins, dtype=np.uint64) // np.uint64(4))[:, None]
    words = np.stack(philox.philox4x32_10(t, blk, 0, 0, k0, k1), axis=0)          # [4, n_bins, T]
    w = np.take_along_axis(words, (np.arange(n_bins) % 4)[None, :, None].repeat(T, axis=2), axis=0)[0]
    u = philox.u01(w).astype(F64)
    return np.exp(2j * np.pi * u).astype(np.complex64)


def griffinlim(S, angles, n_iter, momentum=MOMENTUM, dtype=F32, **cfg):
    """librosa 0.7 griffinlim(S, n_iter, hop_length, win_length) from the initial phases `angles` (complex64;
    dtype=float64: float64 and complex128 throughout)."""
    c = dict(MO.DEFAULT, dtype=dtype, **cfg)
    S = np.asarray(S, dtype)
    angles = np.array(angles, dtype=np.result_type(dtype, 1j))
    rebuilt = 0.0
    for _ in range(n_iter):
        tprev = rebuilt
        inverse = istft(S * angles, **c)
        rebuilt = stft(inverse, **c)
        angles[:] = rebuilt - (momentum / (1 + momentum)) * tprev
        angles[:] /= np.abs(angles) + 1e-16
    return istft(S * angles, **c)


def reconstruct_waveform(mel, n_iter=32, seed=0, solver="fista", **cfg):
    """The whole path: float32 [hop_length * (T - 1)]."""
    c = dict(MO.DEFAULT, **cfg)
    S = mel_to_stft(mel, solver=solver, **c)
    return griffinlim(S, phases(seed, S.shape[1], S.shape[0]), n_iter, **c)


def spectral_convergence(y, S, **cfg):
    """|| |stft(y)| - S || / ||S||, in float64."""
    c = dict(MO.DEFAULT, **cfg)
    got = np.abs(stft(y, **c)).astype(F64)
    return float(np.linalg.norm(got - S) / np.linalg.norm(np.asarray(S, F64)))
