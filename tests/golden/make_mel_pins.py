"""Pins of the mel analysis from an implementation independent of tests/mel_oracle.py (torch's STFT and torchaudio's
Slaney filterbank, both in float64):

    python tests/golden/make_mel_pins.py

writes tests/golden/mel_pins.npz with
  fbank  [80, 1025]  torchaudio.functional.melscale_fbanks(1025, 40, 11025, 80, 22050, norm='slaney',
                     mel_scale='slaney'), transposed
  mel    [80, 164]   normalize(amp_to_db(fbank @ |torch.stft(y, 2048, 275, 1100, hann_window(1100, periodic),
                     center=True, pad_mode='reflect')|)) of the speech waveform in trained_tacotron.npz ('wav')
The arrays depend on torch and torchaudio alone: a second run writes identical arrays."""
from pathlib import Path

import numpy as np
import torch
import torchaudio

HERE = Path(__file__).resolve().parent


def main():
    sr, n_fft, hop, win, n_mels, fmin = 22050, 2048, 275, 1100, 80, 40.0
    y = np.load(HERE / "trained_tacotron.npz")["wav"].astype(np.float32)
    fb = torchaudio.functional.melscale_fbanks(1 + n_fft // 2, fmin, sr / 2, n_mels, sr, norm="slaney",
                                               mel_scale="slaney").T.double()
    D = torch.stft(torch.tensor(y, dtype=torch.float64), n_fft, hop, win,
                   window=torch.hann_window(win, periodic=True, dtype=torch.float64), center=True, pad_mode="reflect",
                   return_complex=True).abs()
    M = fb @ D
    mel = torch.clamp((20 * torch.log10(torch.clamp(M, min=1e-5)) + 100) / 100, 0, 1)
    np.savez_compressed(HERE / "mel_pins.npz", fbank=fb.numpy(), mel=mel.numpy().astype(np.float32))


if __name__ == "__main__":
    main()
