"""The designed grid of the mel analysis edge tests: named configurations of wrnn_mel_create covering each axis it
accepts at its ends and at one odd interior value, the signals each configuration is analysed on, and deliberately
wrong restatements of tests/mel_oracle.py's melspectrogram (same signature) that the tolerance must tell apart.
Shared by tests/test_mel_edges.py (the oracle against tests/golden/mel_pins.npz, the host tables and the kernel's
per-frame code run on the host) and tests/test_gpu_mel_edges.py (the kernel).

Everything is deterministic (fixed seeds); every fmin and min_level_db is exact in float32, as wrnn_mel_cfg stores
them."""
from __future__ import annotations

import numpy as np
import scipy.fft
import scipy.signal

import mel_oracle as MO

F32 = np.float32
# name -> the configuration's keys that differ from mel_oracle.DEFAULT (22,050 Hz, n_fft 2048, hop 275, win 1100,
# 80 mels, fmin 40, -100 dB)
GRID = {
    "default": {},
    "win1": dict(win_length=1),
    "win2": dict(win_length=2),
    "win3": dict(win_length=3),
    "win1101": dict(win_length=1101),
    "win2047": dict(win_length=2047),
    "win2048": dict(win_length=2048),
    # n_fft 256 / 512: fewer butterflies per stage (64 / 128) than the kernel's 256 threads
    "fft256-mels128": dict(n_fft=256, win_length=255, hop_length=200, n_mels=128),
    "fft256-hop1": dict(n_fft=256, win_length=200, hop_length=1),
    "fft512-hop600": dict(n_fft=512, win_length=511, hop_length=600),
    "fft4096-hop5000": dict(n_fft=4096, win_length=3001, hop_length=5000),
    "hop1-fft2048": dict(hop_length=1, n_mels=7),
    "sr8k-fft256-mels128": dict(sample_rate=8000, n_fft=256, win_length=256, hop_length=100, n_mels=128, fmin=0.0),
    "sr16k-fmin2000": dict(sample_rate=16000, n_fft=1024, win_length=800, hop_length=200, fmin=2000.0),
    "sr16k-fmin7990": dict(sample_rate=16000, hop_length=200, win_length=800, fmin=7990.0),
    "sr44k": dict(sample_rate=44100, n_fft=4096, win_length=2200, hop_length=551),
    "sr44k-fmin2000-mels128": dict(sample_rate=44100, n_mels=128, fmin=2000.0, hop_length=441),
    "sr1": dict(sample_rate=1, fmin=0.25),
    "mels1": dict(n_mels=1),
    "mels37-fmin1234.5": dict(n_mels=37, fmin=1234.5),
    "db-20": dict(min_level_db=-20.0),
    "db-37.5": dict(min_level_db=-37.5),
    "db-120": dict(min_level_db=-120.0),
}

# Grid points pinned by torch's STFT and torchaudio's filterbank on the speech fixture (tests/golden/make_mel_pins.py),
# with the sample rate the speech is resampled to (None: the fixture's own 22,050 Hz)
PINS = {"win1": None, "win1101": None, "fft256-mels128": None, "sr16k-fmin2000": 16000, "sr44k": 44100, "db-120": None}


def cfg(name):
    return dict(MO.DEFAULT, **GRID[name])


def signals(c, seed=0):
    """The signals of configuration c (all keys): name -> float32 waveform.  Four shapes of content at a base length of
    about 24 frames (noise, a tone off the bin grid, a chirp across the band, noise at 4x full scale, digital silence
    with one click), then noise at the lengths where the frame count changes: the minimum n_fft / 2 + 1, a multiple of
    hop, one short of a multiple, and (where hop allows it) shorter than one hop, so T = 1."""
    sr, n_fft, hop = c["sample_rate"], c["n_fft"], c["hop_length"]
    rs = np.random.RandomState(seed)
    n = n_fft + 24 * hop + 17
    t = np.arange(n) / sr
    click = np.zeros(n, F32)
    click[n // 2 - 3] = F32(0.99)
    s = {
        "noise": np.clip(0.3 * rs.randn(n), -1, 1).astype(F32),
        "tone": (0.9 * np.sin(2 * np.pi * 0.0234 * sr * t)).astype(F32),
        "chirp": (0.5 * scipy.signal.chirp(t, 0.002 * sr, t[-1], 0.45 * sr)).astype(F32),
        "overdriven": (4 * rs.randn(n)).astype(F32),
        "silence_click": click,
    }
    lo = n_fft // 2 + 1
    mult = hop * (lo // hop + 2)
    lengths = {"min": lo, "mult_hop": mult, "mult_hop-1": mult + hop - 1}
    if hop > lo:
        lengths["under_hop"] = hop - 1
    for k, m in lengths.items():
        if m not in [v.size for v in s.values()]:
            s[k] = np.clip(0.3 * rs.randn(m), -1, 1).astype(F32)
    return s


def silent_value(min_level_db):
    """What a frame of digital silence analyses to: float32(clip((-100 - L) / -L, 0, 1))."""
    L = float(F32(min_level_db))
    return F32(np.clip((-100.0 - L) / -L, 0, 1))


# ---- wrong restatements ----------------------------------------------------------------------------------------------
def _restated(y, *, window=None, pad="reflect", c64=True, fb32=False, sum32=False, log32=False, **cfg):
    """melspectrogram with one step done wrong; the defaults restate mel_oracle.melspectrogram."""
    c = dict(MO.DEFAULT, **cfg)
    n_fft, hop = c["n_fft"], c["hop_length"]
    yp = np.pad(np.asarray(y, F32), n_fft // 2, mode=pad)
    T = 1 + (len(yp) - n_fft) // hop
    w = MO.window(**c) if window is None else window(**c)
    frames = yp[np.arange(n_fft)[:, None] + hop * np.arange(T)[None]].astype(np.float64)
    X = scipy.fft.rfft(w[:, None] * frames, axis=0)
    mag = (np.abs(X.astype(np.complex64)) if c64 else np.abs(X)).astype(np.float64)
    fb = MO.mel_basis(**c)
    if fb32:
        fb = fb.astype(F32).astype(np.float64)
    M = (fb.astype(F32) @ mag.astype(F32)).astype(np.float64) if sum32 else fb @ mag
    if log32:
        S = (F32(20) * np.log10(np.maximum(F32(1e-5), M.astype(F32)))).astype(np.float64)
    else:
        S = 20 * np.log10(np.maximum(1e-5, M))
    return np.clip((S - c["min_level_db"]) / -c["min_level_db"], 0, 1).astype(F32)


def _symmetric_window(n_fft, win_length, **_):
    w = scipy.signal.get_window("hann", win_length, fftbins=False)
    lp = (n_fft - win_length) // 2
    return np.pad(w, (lp, n_fft - win_length - lp))


# the visible slips: each must miss the kernel's tolerance (test_mel_abi.MEL_TOL) in at least one cell of the grid
WRONG = {
    "window_one_sample_off": lambda y, **c: _restated(y, window=lambda **k: np.roll(MO.window(**k), 1), **c),
    "symmetric_window": lambda y, **c: _restated(y, window=_symmetric_window, **c),
    "symmetric_padding": lambda y, **c: _restated(y, pad="symmetric", **c),
    "float32_window": lambda y, **c: _restated(y, window=lambda **k: MO.window(**k).astype(F32).astype(np.float64), **c),
    "float32_log10": lambda y, **c: _restated(y, log32=True, **c),
    "float32_fft": lambda y, **c: MO.melspectrogram(y, fft_dtype=np.float32, **c),
    "float32_band_sums": lambda y, **c: _restated(y, sum32=True, **c),
}
# slips the output cannot show: their gaps stay inside the tolerance (they sit below the output's own rounding)
INVISIBLE = {
    "no_complex64_rounding": lambda y, **c: _restated(y, c64=False, **c),
    "float32_filterbank": lambda y, **c: _restated(y, fb32=True, **c),
}
