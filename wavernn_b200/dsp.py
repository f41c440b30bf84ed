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


def _analysis():
    """The analysis object for hp's sample_rate, n_fft, hop_length, win_length, num_mels, fmin and min_level_db."""
    from . import cabi
    key = (hp.sample_rate, hp.n_fft, hp.hop_length, hp.win_length, hp.num_mels, hp.fmin, hp.min_level_db)
    if key not in _analyses:
        _analyses[key] = cabi.MelAnalysis(sample_rate=hp.sample_rate, n_fft=hp.n_fft, hop_length=hp.hop_length,
                                          win_length=hp.win_length, n_mels=hp.num_mels, fmin=hp.fmin,
                                          min_level_db=hp.min_level_db)
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
    seed = int(np.random.randint(0, 2 ** 63 - 1, dtype=np.int64))
    return _analysis().griffinlim_many_host([mel], n_iter, [seed])[0]


def save_wav(x, path, sample_rate=None):
    """float32 wav at hp.sample_rate (utils/dsp.py:22-23 wrote through
    librosa.output.write_wav, removed in librosa>=0.8)."""
    from scipy.io import wavfile
    sr = int(sample_rate if sample_rate is not None else hp.sample_rate)
    wavfile.write(str(path), sr, np.asarray(x).astype(np.float32))
