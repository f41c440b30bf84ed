"""numpy restatement of the reference's melspectrogram(y) (utils/dsp.py:72-81) through librosa 0.6.3: the periodic Hann
window centred in n_fft, reflect padding, a float64 FFT rounded to complex64 (stft(dtype=np.complex64)), abs, the
float64 Slaney filterbank with Slaney norm (filters.mel, htk=False, norm=1), amp_to_db and normalize -- and of the
targets preprocess.py stores (float32, as numpy 1.22 evaluates them), mapped back with label_2_float."""
import numpy as np
import scipy.fft
import scipy.signal

DEFAULT = dict(sample_rate=22050, n_fft=2048, hop_length=275, win_length=1100, n_mels=80, fmin=40.0, min_level_db=-100.0)
F32 = np.float32


def hz_to_mel(f):
    f = np.asanyarray(f, dtype=np.float64)
    f_sp, min_log_hz = 200.0 / 3, 1000.0
    min_log_mel, logstep = min_log_hz / f_sp, np.log(6.4) / 27.0
    return np.where(f >= min_log_hz, min_log_mel + np.log(np.maximum(f, min_log_hz) / min_log_hz) / logstep, f / f_sp)


def mel_to_hz(m):
    m = np.asanyarray(m, dtype=np.float64)
    f_sp, min_log_hz = 200.0 / 3, 1000.0
    min_log_mel, logstep = min_log_hz / f_sp, np.log(6.4) / 27.0
    return np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), f_sp * m)


def mel_basis(sample_rate, n_fft, n_mels, fmin, **_):
    """librosa 0.6.3 filters.mel(sr, n_fft, n_mels, fmin), fmax = sr / 2, in float64: [n_mels, n_fft // 2 + 1]."""
    fft = np.linspace(0, sample_rate / 2, 1 + n_fft // 2, endpoint=True)
    mel_f = mel_to_hz(np.linspace(hz_to_mel(fmin), hz_to_mel(sample_rate / 2), n_mels + 2))
    fdiff, ramps = np.diff(mel_f), np.subtract.outer(mel_f, fft)
    w = np.zeros((n_mels, 1 + n_fft // 2))
    for i in range(n_mels):
        w[i] = np.maximum(0, np.minimum(-ramps[i] / fdiff[i], ramps[i + 2] / fdiff[i + 1]))
    return w * (2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels]))[:, None]


def window(n_fft, win_length, **_):
    """scipy.signal.get_window('hann', win_length, fftbins=True) padded as librosa.util.pad_center: [n_fft] float64."""
    w = scipy.signal.get_window("hann", win_length, fftbins=True)
    lp = (n_fft - win_length) // 2
    return np.pad(w, (lp, n_fft - win_length - lp))


def magnitudes(y, *, n_fft, hop_length, win_length, fft_dtype=np.float64, chunk=4096, **_):
    """|stft(y)| as librosa 0.6.3 stores it (complex64), [n_fft // 2 + 1, 1 + len(y) // hop_length] float32."""
    y = np.asarray(y, dtype=np.float32)
    yp = np.pad(y, n_fft // 2, mode="reflect")
    T = 1 + (len(yp) - n_fft) // hop_length
    win = window(n_fft, win_length).astype(fft_dtype)
    out = np.empty((n_fft // 2 + 1, T), dtype=np.float32)
    for t0 in range(0, T, chunk):
        t = np.arange(t0, min(T, t0 + chunk))
        frames = yp[np.arange(n_fft)[:, None] + hop_length * t[None]].astype(fft_dtype)
        out[:, t] = np.abs(scipy.fft.rfft(win[:, None] * frames, axis=0).astype(np.complex64))
    return out


def melspectrogram(y, fft_dtype=np.float64, **cfg):
    """melspectrogram(y) for the configuration `cfg` (DEFAULT's keys): float32 [n_mels, 1 + len(y) // hop_length].
    fft_dtype=np.float32 gives the single-precision transform (the negative control of the kernel's tolerance)."""
    c = dict(DEFAULT, **cfg)
    M = mel_basis(**c) @ magnitudes(y, fft_dtype=fft_dtype, **c).astype(np.float64)
    S = 20 * np.log10(np.maximum(1e-5, M))
    return np.clip((S - c["min_level_db"]) / -c["min_level_db"], 0, 1).astype(np.float32)


# ---- the targets of wrnn_score_wav_many ------------------------------------------------------------------------------
def normalise(y, peak_norm):
    """preprocess.py:38-40: y / max|y| (float32) when peak_norm is set or the peak exceeds 1."""
    y = np.asarray(y, dtype=F32)
    peak = np.abs(y).max()
    return y / peak if peak_norm or peak > 1.0 else y


def labels(y, mode, bits=9, mu_law=False):
    """preprocess.py:41-45 in float32: the stored int64 labels."""
    y = np.asarray(y, dtype=F32)
    if mode == "RAW" and mu_law:
        mu = F32(2 ** bits - 1)
        fx = np.sign(y) * np.log(F32(1) + mu * np.abs(y)) / F32(np.log(2.0 ** bits))
        return np.floor((fx + F32(1)) / F32(2) * mu + F32(0.5)).astype(np.int64)
    b = 16 if mode == "MOL" else bits
    top = F32(2 ** b - 1)
    return np.clip((y + F32(1)) * top / F32(2), F32(0), top).astype(np.int64)


def targets(y, mode, bits=9, mu_law=False):
    """utils/dataset.py:86-91: label_2_float of the labels, in float32 as torch evaluates it."""
    b = 16 if mode == "MOL" else bits
    return (F32(2) * labels(y, mode, bits, mu_law).astype(F32)) / F32(2 ** b - 1) - F32(1)


# ---- signals ---------------------------------------------------------------------------------------------------------
def signals(sr=22050, seconds=2.0, seed=0):
    """The test signals at sample rate sr: name -> float32 waveform."""
    rs = np.random.RandomState(seed)
    t = np.arange(int(sr * seconds)) / sr
    click = np.zeros(t.size)
    click[t.size // 2 - 3] = 0.99
    return {
        "tone440": (0.9 * np.sin(2 * np.pi * 440 * t)).astype(F32),
        "chirp": (0.5 * scipy.signal.chirp(t, 40, t[-1], 11000)).astype(F32),
        "noise_full": np.clip(rs.randn(t.size), -1, 1).astype(F32),
        "noise_1e-4": (1e-4 * rs.randn(t.size)).astype(F32),
        "silence_click": click.astype(F32),
    }
