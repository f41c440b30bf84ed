"""wrnn_griffinlim_many on the GPU.

  1. The kernels against the host run of their code (wrnn_debug_griffinlim) and the oracle (tests/gl_oracle.py) at
     every configuration of test_gl_abi.GL_CONFIGS: n_iter = 0 pins S (the solve) and the inverse transform, since that
     output is linear in S; n_iter = 1 adds one phase update.
  2. The 16 Tacotron mels in one batch at 32 iterations against the oracle (test_gl_abi.GL32_TOL), and the quality of
     the reconstruction: spectral convergence falls with the iterations and ends at or below 0.2, and the analysis of
     the output lands near the input mel.
  3. A batch of mixed lengths (the minimum T included) is bit-identical to each mel alone, the host entry to the device
     entry, a seed to itself; a NaN mel leaves the rest of its batch bit-identical.
  4. wavernn_b200.dsp.reconstruct_waveform is repeatable under np.random.seed.
Run on a GPU: pytest -m gpu -s tests/test_gpu_griffinlim.py"""
import numpy as np
import pytest
import torch

import gl_oracle as G
import helpers
import mel_oracle as MO
from test_gl_abi import GL32_TOL, GL_CONFIGS, ULPS_EARLY, config_mel, host_gl
from wavernn_b200 import cabi

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
# the analysis of the 32-iteration output against the input mel, in normalized units: over the 16 Tacotron mels the
# oracle gives a median of at most 0.0055 and a 99th percentile of 0.052-0.065, except the two shortest mels (164 and
# 98 frames: 0.089 and 0.094, their edge frames weigh more)
RT_MEDIAN, RT_P99 = 0.01, 0.12


def gl_device(an, mels, seeds, n_iter):
    """wrnn_griffinlim_many on device copies of mels (one batch); returns the host waveforms."""
    dm = [torch.as_tensor(np.ascontiguousarray(m, dtype=np.float32), device=DEV) for m in mels]
    dw = [torch.full((an.samples(m.shape[1]),), float("nan"), device=DEV) for m in mels]
    an.griffinlim_many(mels=[m.data_ptr() for m in dm], Ts=[m.shape[1] for m in mels], seeds=seeds,
                       wavs=[w.data_ptr() for w in dw], n_iter=n_iter, stream=torch.cuda.current_stream(DEV).cuda_stream)
    torch.cuda.synchronize(DEV)
    return [w.cpu().numpy() for w in dw]


@pytest.mark.parametrize("name", list(GL_CONFIGS))
def test_kernels_against_host_run_and_oracle(name):
    lib = cabi.load()
    mel, c = config_mel(name)
    an = cabi.MelAnalysis(**GL_CONFIGS[name])
    try:
        S_ref = G.mel_to_stft(mel, **c)
        for n_iter in (0, 1):
            got = gl_device(an, [mel], [7], n_iter)[0]
            host, _ = host_gl(lib, mel, 7, n_iter, **c)
            ref = G.griffinlim(S_ref, G.phases(7, S_ref.shape[1], S_ref.shape[0]), n_iter, **c)
            step = np.spacing(np.abs(ref).max())
            d_ref, d_host = np.abs(got - ref).max() / step, np.abs(got - host).max() / step
            print(f"{name} n_iter={n_iter}: device vs oracle {d_ref:.1f}, vs host run {d_host:.1f} float32 steps of the peak")
            assert got.shape == ref.shape and np.isfinite(got).all()
            assert d_ref <= ULPS_EARLY and d_host <= ULPS_EARLY
    finally:
        an.close()


def test_tacotron_mels_32_iterations_and_quality():
    an = cabi.MelAnalysis()
    try:
        mels = helpers.tacotron_mels()
        seeds = list(range(100, 116))
        outs = {n: gl_device(an, mels, seeds, n) for n in (0, 8, 32)}
        worst, rts = 0.0, []
        for i, mel in enumerate(mels):
            S = G.mel_to_stft(mel)
            ref = G.griffinlim(S, G.phases(seeds[i], S.shape[1], S.shape[0]), 32)
            worst = max(worst, float(np.abs(outs[32][i] - ref).max()))
            sc = [G.spectral_convergence(outs[n][i], S) for n in (0, 8, 32)]
            assert sc[0] > sc[1] > sc[2] and sc[2] <= 0.2, (i, sc)
            back = an.melspectrogram_many_host([outs[32][i]])[0]
            assert back.shape == mel.shape
            d = np.abs(back - mel)
            rts.append((float(np.median(d)), float(np.percentile(d, 99))))
            print(f"mel_{i:02d}: spectral convergence {sc[0]:.3f} -> {sc[1]:.3f} -> {sc[2]:.3f}; round trip median "
                  f"{rts[-1][0]:.4f} p99 {rts[-1][1]:.4f}")
        print(f"32 iterations: device vs oracle {worst:.2e} (tolerance {GL32_TOL})")
        assert worst <= GL32_TOL
        assert max(r[0] for r in rts) <= RT_MEDIAN and max(r[1] for r in rts) <= RT_P99
    finally:
        an.close()


def test_batch_equals_single_host_and_repeats():
    an = cabi.MelAnalysis()
    try:
        taco = helpers.tacotron_mels()
        mels = [taco[15][:, :5], taco[0], taco[9][:, :37], taco[3], taco[8][:, :6]]   # T = 5 is the minimum
        seeds = [1, 2, 3, 2 ** 63 + 5, 1]
        batch = gl_device(an, mels, seeds, 4)
        for i, m in enumerate(mels):
            assert batch[i].shape == (275 * (m.shape[1] - 1),) and np.isfinite(batch[i]).all(), i
            assert np.array_equal(gl_device(an, [m], [seeds[i]], 4)[0], batch[i]), i
        assert all(np.array_equal(a, b) for a, b in zip(an.griffinlim_many_host(mels, 4, seeds), batch))
        assert all(np.array_equal(a, b) for a, b in zip(gl_device(an, mels, seeds, 4), batch))
        assert not np.array_equal(gl_device(an, [mels[1]], [99], 4)[0], batch[1])
        bad = mels[1].copy()
        bad[10, 40] = np.nan
        poisoned = gl_device(an, [mels[0], bad, mels[2]], seeds[:3], 4)
        assert np.isnan(poisoned[1]).any()
        assert np.array_equal(poisoned[0], batch[0]) and np.array_equal(poisoned[2], batch[2])
    finally:
        an.close()


def test_reconstruct_waveform_follows_numpy_seed(monkeypatch):
    from wavernn_b200 import dsp
    from wavernn_b200.hp import DEFAULT_HPARAMS_FILE, _HParams
    monkeypatch.setattr(dsp, "hp", _HParams(DEFAULT_HPARAMS_FILE))   # the shipped hparams, leaving the global unset
    mel = helpers.tacotron_mels()[15]
    np.random.seed(5)
    a = dsp.reconstruct_waveform(mel, n_iter=2)
    np.random.seed(5)
    b = dsp.reconstruct_waveform(mel, n_iter=2)
    c = dsp.reconstruct_waveform(mel, n_iter=2)
    assert a.dtype == np.float32 and a.shape == (275 * (mel.shape[1] - 1),)
    assert np.array_equal(a, b) and not np.array_equal(a, c)
