"""Pins of the mel analysis from an implementation independent of tests/mel_oracle.py (torch's STFT and torchaudio's
Slaney filterbank, both in float64):

    python tests/golden/make_mel_pins.py

writes tests/golden/mel_pins.npz with
  fbank  [80, 1025]  torchaudio.functional.melscale_fbanks(1025, 40, 11025, 80, 22050, norm='slaney',
                     mel_scale='slaney'), transposed
  mel    [80, 164]   normalize(amp_to_db(fbank @ |torch.stft(y, 2048, 275, 1100, hann_window(1100, periodic),
                     center=True, pad_mode='reflect')|)) of the speech waveform in trained_tacotron.npz ('wav')
and, for each grid point of tests/mel_edges.py's PINS (its configuration copied below), the same computation at that
configuration: fbank_<name> (float32, as torchaudio builds it), mel_<name> and, where the point's sample rate is not
22,050 Hz, y_<name>, the float32 waveform analysed (the first EXCERPT samples of the speech, resampled by
torchaudio.functional.resample in float64);
window_win1 [2048] is
torch.hann_window(1, periodic=True) centred in n_fft as torch.stft pads it.
The arrays depend on torch and torchaudio alone: a second run writes identical arrays."""
import warnings
from pathlib import Path

import numpy as np
import torch
import torchaudio

HERE = Path(__file__).resolve().parent
DEFAULT = dict(sample_rate=22050, n_fft=2048, hop_length=275, win_length=1100, n_mels=80, fmin=40.0, min_level_db=-100.0)
EXCERPT = 16384   # the speech samples resampled for another sample rate (0.74 s, to keep the fixture small)
# tests/mel_edges.py GRID[name] for each name of PINS
POINTS = {
    "win1": dict(win_length=1),
    "win1101": dict(win_length=1101),
    "fft256-mels128": dict(n_fft=256, win_length=255, hop_length=200, n_mels=128),
    "sr16k-fmin2000": dict(sample_rate=16000, n_fft=1024, win_length=800, hop_length=200, fmin=2000.0),
    "sr44k": dict(sample_rate=44100, n_fft=4096, win_length=2200, hop_length=551),
    "db-120": dict(min_level_db=-120.0),
}


def analyse(y, sample_rate, n_fft, hop_length, win_length, n_mels, fmin, min_level_db):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")   # torchaudio warns about bands without a bin
        fb = torchaudio.functional.melscale_fbanks(1 + n_fft // 2, fmin, sample_rate / 2, n_mels, sample_rate,
                                                   norm="slaney", mel_scale="slaney").T.double()
    D = torch.stft(torch.tensor(y, dtype=torch.float64), n_fft, hop_length, win_length,
                   window=torch.hann_window(win_length, periodic=True, dtype=torch.float64), center=True,
                   pad_mode="reflect", return_complex=True).abs()
    M = fb @ D
    mel = torch.clamp((20 * torch.log10(torch.clamp(M, min=1e-5)) - min_level_db) / -min_level_db, 0, 1)
    return fb.numpy(), mel.numpy().astype(np.float32)


def main():
    y = np.load(HERE / "trained_tacotron.npz")["wav"].astype(np.float32)
    fb, mel = analyse(y, **DEFAULT)
    out = dict(fbank=fb, mel=mel)
    for name, kw in POINTS.items():
        c = dict(DEFAULT, **kw)
        yc = y
        if c["sample_rate"] != DEFAULT["sample_rate"]:
            yc = torchaudio.functional.resample(torch.tensor(y[:EXCERPT], dtype=torch.float64), DEFAULT["sample_rate"],
                                                c["sample_rate"]).numpy().astype(np.float32)
        fb, out[f"mel_{name}"] = analyse(yc, **c)
        out[f"fbank_{name}"] = fb.astype(np.float32)       # torchaudio builds it in float32: stored exactly
        if yc is not y:
            out[f"y_{name}"] = yc
    w = torch.hann_window(1, periodic=True, dtype=torch.float64)
    out["window_win1"] = torch.nn.functional.pad(w, ((2048 - 1) // 2, 2048 - 1 - (2048 - 1) // 2)).numpy()
    np.savez_compressed(HERE / "mel_pins.npz", **out)


if __name__ == "__main__":
    main()
