"""Stand-in for the reference's utils/dsp.py, which imports librosa on its first line.

`python -m wavernn_b200.dropin` serves this file as `utils.dsp` when librosa cannot be imported; the file swap copies
dropin/utils/dsp.py (a re-export of this module) over the checkout's utils/dsp.py.  It is executed when the script
first imports `utils.dsp`, inside the reference checkout, so `hp` is the checkout's own `utils.hparams` singleton,
configured by the script (hp.configure) before any of these functions reads it.  Importing it starts no CUDA context;
load_wav (at another rate), melspectrogram and reconstruct_waveform open one on their first call.

It exports what the scripts read through `from utils.dsp import *`: hp, np and math themselves, the wav I/O, the mel
analysis and Griffin-Lim, the label, mu-law, 16-bit and emphasis helpers, and the dB conversions.  stft, spectrogram
and linear_to_mel are not provided: no script calls them.
"""
import math  # noqa: F401  (exported: the scripts use it through the star import)

import numpy as np
from scipy.signal import lfilter

from utils import hparams as hp
from wavernn_b200 import dsp as _dsp
from wavernn_b200.dsp import decode_mu_law, encode_mu_law, float_2_label, label_2_float  # noqa: F401


def load_wav(path):
    """librosa.load(path, sr=hp.sample_rate)[0] for WAV files (wavernn_b200.dsp.load_wav with this checkout's hp)."""
    return _dsp._load_wav(path, hp)


def save_wav(x, path):
    """x as a float32 WAV at hp.sample_rate."""
    _dsp.save_wav(x, path, hp.sample_rate)


def split_signal(x):
    """A 16-bit signal as (coarse, fine) bytes of its offset-binary value."""
    u = x + 2 ** 15
    return u // 256, u % 256


def combine_signal(coarse, fine):
    return (coarse * 256 + fine) - 2 ** 15


def encode_16bits(x):
    return np.clip(x * 2 ** 15, -2 ** 15, 2 ** 15 - 1).astype(np.int16)


def amp_to_db(x):
    return 20 * np.log10(np.maximum(1e-5, x))


def db_to_amp(x):
    return np.power(10.0, x * 0.05)


def normalize(S):
    """dB relative to hp.min_level_db, mapped to [0, 1]."""
    return np.clip((S - hp.min_level_db) / -hp.min_level_db, 0, 1)


def denormalize(S):
    return np.clip(S, 0, 1) * -hp.min_level_db + hp.min_level_db


def melspectrogram(y):
    """The normalized mel of y with hp's analysis fields, on the device: float32 [num_mels, 1 + len(y) // hop_length]."""
    return _dsp._analysis(hp).melspectrogram_many_host([y])[0]


def reconstruct_waveform(mel, n_iter=32):
    """Griffin-Lim from a normalized mel with hp's analysis fields, on the device (wavernn_b200.dsp.reconstruct_waveform
    with this checkout's hp)."""
    return _dsp._reconstruct(mel, n_iter, hp)


def pre_emphasis(x):
    """y[t] = x[t] - hp.preemphasis * x[t - 1]."""
    return lfilter([1, -hp.preemphasis], [1], x)


def de_emphasis(x):
    """The inverse filter of pre_emphasis."""
    return lfilter([1], [1, -hp.preemphasis], x)
