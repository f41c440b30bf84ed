"""wrnn_resample_many on the GPU.

  1. The kernel against its host run (wrnn_debug_resample) and the oracle (tests/resample_oracle.py) at every rate of
     test_resample_abi.RATES, on tones, a chirp, noise and a speech-like signal, and at the edge lengths: bit-identical.
  2. A mixed-rate batch is bit-identical to each utterance alone, the host entry to the device entry; nothing is written
     past wrnn_resample_length; a NaN utterance leaves the rest of its batch bit-identical.
  3. End to end: dsp.load_wav of a 44.1 kHz WAV, then melspectrogram, against the mel of the same signal synthesised at
     22,050 Hz; and the drop-in's utils.dsp stand-in running load_wav -> melspectrogram on a 48 kHz file.
Run on a GPU: pytest -m gpu -s tests/test_gpu_resample.py"""
import importlib.util

import numpy as np
import pytest
import torch

import resample_oracle as R
from test_dropin_dsp import make_checkout, run_dropin, write_wav16
from test_resample_abi import RATES, SR, host, same_bits, signals
from wavernn_b200 import cabi, dsp

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
SENTINEL = 7.0


@pytest.fixture(scope="module")
def an():
    a = cabi.MelAnalysis()
    yield a
    a.close()


@pytest.fixture(scope="module")
def lib():
    return cabi.load()


@pytest.fixture(scope="module")
def win(lib):
    w = np.empty(lib.wrnn_debug_resample_table(None), dtype=np.float64)
    lib.wrnn_debug_resample_table(w.ctypes.data)
    return w


def device(an, xs, rates, stream=None):
    """wrnn_resample_many on device copies (one batch); each output is followed by a sentinel that must survive."""
    dx = [torch.as_tensor(np.ascontiguousarray(x, dtype=np.float32), device=DEV) for x in xs]
    dy = [torch.full((an.resample_length(x.size, r) + 1,), SENTINEL, device=DEV) for x, r in zip(xs, rates)]
    st = stream or torch.cuda.current_stream(DEV)
    an.resample_many(xs=[x.data_ptr() for x in dx], ns=[x.numel() for x in dx], rates=rates,
                     ys=[y.data_ptr() for y in dy], stream=st.cuda_stream)
    torch.cuda.synchronize(DEV)
    out = [y.cpu().numpy() for y in dy]
    assert all(y[-1] == SENTINEL for y in out), "written past wrnn_resample_length"
    return [y[:-1] for y in out]


@pytest.mark.parametrize("sr", RATES)
def test_device_matches_host_run_and_oracle(an, lib, win, sr):
    sig = signals(sr, sr)
    got = device(an, list(sig.values()), [sr] * len(sig))
    hosted = host(lib, list(sig.values()), [sr] * len(sig))
    for (name, x), y, h in zip(sig.items(), got, hosted):
        assert same_bits(y, h), f"{name} at {sr} Hz: device vs host run"
        assert same_bits(y, R.resample(x, sr, SR, win=win)), f"{name} at {sr} Hz: device vs oracle"


def test_edge_lengths(an, lib):
    cases = [(8000, 1), (16000, 1), (44100, 2), (48000, 3), (16000, 40), (48000, 200), (44100, 127), (44100, 1001),
             (8000, 63), (22051, 5), (22050, 1)]
    xs = [np.random.RandomState(n).uniform(-1, 1, n).astype(np.float32) for _, n in cases]
    rates = [sr for sr, _ in cases]
    for x, y, h in zip(xs, device(an, xs, rates), host(lib, xs, rates)):
        assert same_bits(y, h)


def test_mixed_batch_is_each_alone_and_host_entry(an):
    rs = np.random.RandomState(5)
    rates = [44100, 48000, 16000, 8000, 24000, 22051, 22050, 48000, 44100, 96000]
    xs = [signals(sr, int(sr * rs.uniform(0.2, 1.5)), seed=i)["speech"] for i, sr in enumerate(rates)]
    batch = device(an, xs, rates)
    for i, (x, sr) in enumerate(zip(xs, rates)):
        assert same_bits(batch[i], device(an, [x], [sr])[0]), f"utterance {i} at {sr} Hz"
    via_host = an.resample_many_host(xs, rates)
    for i, (a, b) in enumerate(zip(batch, via_host)):
        assert same_bits(a, b), f"utterance {i}: host entry"


def test_two_streams_share_the_object(an):
    xs = [signals(sr, sr, seed=2)["noise"] for sr in (44100, 48000)]
    want = device(an, xs, [44100, 48000])
    s1, s2 = torch.cuda.Stream(DEV), torch.cuda.Stream(DEV)
    assert all(same_bits(a, b) for a, b in zip(device(an, xs[:1], [44100], s1) + device(an, xs[1:], [48000], s2), want))


def test_nan_utterance_is_isolated(an):
    rates = [44100, 48000, 16000]
    xs = [signals(sr, sr // 2, seed=9)["tones"] for sr in rates]
    alone = device(an, xs, rates)
    bad = xs[1].copy()
    bad[len(bad) // 2] = np.nan
    got = device(an, [xs[0], bad, xs[2]], rates)
    assert same_bits(got[0], alone[0]) and same_bits(got[2], alone[2])
    assert np.isnan(got[1]).any()


def harmonics(sr, secs=2.0):
    """150 Hz and its harmonics up to 4.95 kHz under a slow envelope."""
    t = np.arange(int(sr * secs)) / sr
    return (0.5 + 0.4 * np.sin(2 * np.pi * 1.3 * t)) * sum(0.25 / k * np.sin(2 * np.pi * 150 * k * t + k) for k in range(1, 34))


# load_wav -> melspectrogram of a 44.1 kHz WAV against the mel of the same signal made at 22,050 Hz, frames 5 .. T - 6
# (the first and last 5 frames see the recording's abrupt ends, where the two signals differ): measured 1.2e-5 for a
# float WAV and 0.042 for 16-bit PCM, whose quantisation noise sets the quiet bands above 5 kHz
E2E_TOL = {"float32": 5e-5, "int16": 0.06}


@pytest.mark.parametrize("kind", ["float32", "int16"])
def test_load_wav_then_mel(tmp_path, monkeypatch, kind):
    from scipy.io import wavfile

    from wavernn_b200.hp import DEFAULT_HPARAMS_FILE, _HParams
    monkeypatch.setattr(dsp, "hp", _HParams(DEFAULT_HPARAMS_FILE))   # the shipped hparams, leaving the global unset
    x = harmonics(44100)
    data = x.astype(np.float32) if kind == "float32" else np.round(x * 32767).astype(np.int16)
    wavfile.write(str(tmp_path / "a.wav"), 44100, data)
    y = dsp.load_wav(tmp_path / "a.wav")
    ref = harmonics(SR).astype(np.float32)
    assert y.dtype == np.float32 and y.size == ref.size
    d = np.abs(dsp.melspectrogram(y) - dsp.melspectrogram(ref))[:, 5:-5]
    print(f"load_wav({kind} 44.1 kHz) -> mel vs 22.05 kHz synthesis: max {d.max():.3e}, mean {d.mean():.3e}")
    assert d.max() <= E2E_TOL[kind]


@pytest.mark.skipif(importlib.util.find_spec("librosa") is not None, reason="librosa is importable: no stand-in")
def test_dropin_script_resamples_and_analyses(tmp_path, an):
    make_checkout(tmp_path)
    rs = np.random.RandomState(4)
    x = np.round(harmonics(48000, 1.0) * 30000 + rs.randn(48000) * 30).astype(np.int16)
    write_wav16(tmp_path / "b.wav", x[:, None], 48000)
    out = run_dropin(tmp_path, "mel", str(tmp_path / "b.wav"))
    assert out["standin"] == "standin"
    y, mel = np.load(tmp_path / "loaded.npy"), np.load(tmp_path / "mel.npy")
    want = an.resample_many_host([x.astype(np.float32) * (1.0 / 32768)], [48000])[0]
    assert same_bits(y, want)
    assert y.size == an.resample_length(48000, 48000) == 22050
    assert same_bits(mel, an.melspectrogram_many_host([want])[0])
