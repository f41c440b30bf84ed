"""Host-side DSP helpers on the generate() epilogue (reference utils/dsp.py:8-23,
92-103).  librosa is not a dependency: wavs are written with scipy."""
import math

import numpy as np

from .hp import hparams as hp


def label_2_float(x, bits):
    return 2 * x / (2 ** bits - 1.) - 1.


def float_2_label(x, bits):
    assert abs(x).max() <= 1.0
    x = (x + 1.) * (2 ** bits - 1) / 2
    return x.clip(0, 2 ** bits - 1)


def encode_mu_law(x, mu):
    mu = mu - 1
    fx = np.sign(x) * np.log(1 + mu * np.abs(x)) / np.log(1 + mu)
    return np.floor((fx + 1) / 2 * mu + 0.5)


def decode_mu_law(y, mu, from_labels=True):
    """utils/dsp.py:98-103."""
    if from_labels:
        y = label_2_float(y, math.log2(mu))
    mu = mu - 1
    return np.sign(y) / mu * ((1 + mu) ** np.abs(y) - 1)


_analyses = {}


def _analysis(h=None):
    """The analysis object for h's sample_rate, n_fft, hop_length, win_length, num_mels, fmin and min_level_db (h:
    this package's hparams, or the reference checkout's own for the utils.dsp stand-in)."""
    from . import cabi
    h = hp if h is None else h
    key = (h.sample_rate, h.n_fft, h.hop_length, h.win_length, h.num_mels, h.fmin, h.min_level_db)
    if key not in _analyses:
        _analyses[key] = cabi.MelAnalysis(sample_rate=h.sample_rate, n_fft=h.n_fft, hop_length=h.hop_length,
                                          win_length=h.win_length, n_mels=h.num_mels, fmin=h.fmin,
                                          min_level_db=h.min_level_db)
    return _analyses[key]


def melspectrogram(y):
    """utils/dsp.py:melspectrogram(y) with hp's sample_rate, n_fft, hop_length, win_length, num_mels, fmin and
    min_level_db, computed on the device (wrnn_melspectrogram_many_host; there is no CPU path): float32 [num_mels,
    1 + len(y) // hop_length]."""
    return _analysis().melspectrogram_many_host([y])[0]


def reconstruct_waveform(mel, n_iter=32):
    """utils/dsp.py:reconstruct_waveform(mel, n_iter): Griffin-Lim from a normalized mel [num_mels, T] with the same hp
    fields as melspectrogram, on the device (wrnn_griffinlim_many_host; there is no CPU path): float32
    [hop_length * (T - 1)].  The initial phases are keyed by a draw from numpy's global generator, so np.random.seed
    makes the result repeatable, as it does for the reference's librosa.griffinlim."""
    return _reconstruct(mel, n_iter, hp)


def _reconstruct(mel, n_iter, h):
    seed = int(np.random.randint(0, 2 ** 63 - 1, dtype=np.int64))
    return _analysis(h).griffinlim_many_host([mel], n_iter, [seed])[0]


def read_wav(path):
    """A WAV file as load_wav decodes it, before resampling: (float32 mono samples, sample rate).  16-bit PCM becomes
    int16 * 2^-15 in float32 and channels are averaged in float32 (np.mean), both as librosa 0.6.3 does.  Departure:
    the other encodings scipy reads (8-, 24- and 32-bit PCM, float) are scaled to [-1, 1] at full precision, where
    librosa 0.6.3 decodes them through audioread.  Anything that is not a WAV file is refused (ValueError)."""
    from scipy.io import wavfile
    try:
        sr, data = wavfile.read(str(path))
    except ValueError as e:
        raise ValueError(f"load_wav: {path} is not a WAV file scipy can read ({e})") from None
    if data.dtype == np.int16:
        y = data.astype(np.float32) * (1.0 / 32768)
    elif data.dtype == np.uint8:
        y = ((data.astype(np.float64) - 128) / 128).astype(np.float32)
    elif data.dtype == np.int32:                       # 24- and 32-bit PCM, left-aligned in int32
        y = (data / 2.0 ** 31).astype(np.float32)
    elif data.dtype.kind == "f":
        y = data.astype(np.float32)
    else:
        raise ValueError(f"load_wav: {path}: unsupported WAV sample type {data.dtype}")
    if y.ndim > 1:
        y = np.mean(y.T, axis=0)
    return np.ascontiguousarray(y, dtype=np.float32), int(sr)


def load_wav(path):
    """utils/dsp.py:load_wav(path): librosa.load(path, sr=hp.sample_rate) (librosa 0.6.3) for WAV files: read_wav, then,
    when the file's rate is not hp.sample_rate, resampy's kaiser_best resampling on the device
    (MelAnalysis.resample_many_host; there is no CPU path).  A file already at hp.sample_rate needs no GPU.  float32
    [ceil(n * hp.sample_rate / rate)]."""
    return _load_wav(path, hp)


def _load_wav(path, h):
    y, sr = read_wav(path)
    if sr == int(h.sample_rate):
        return y
    return _analysis(h).resample_many_host([y], [sr])[0]


def save_wav(x, path, sample_rate=None):
    """float32 wav at hp.sample_rate (utils/dsp.py:22-23 wrote through
    librosa.output.write_wav, removed in librosa>=0.8)."""
    from scipy.io import wavfile
    sr = int(sample_rate if sample_rate is not None else hp.sample_rate)
    wavfile.write(str(path), sr, np.asarray(x).astype(np.float32))
