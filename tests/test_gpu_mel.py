"""wrnn_melspectrogram_many and wrnn_score_wav_many on the GPU.

  1. The kernel against tests/mel_oracle.py, one absolute tolerance (test_mel_abi.MEL_TOL, 2^-23: one output step)
     for every signal -- the checkpoint's vocoded speech, a 440 Hz tone, a chirp, full-scale and 1e-4 noise, digital
     silence with one click (silent frames exactly 0), the minimum length, ten minutes -- and every configuration.
  2. A batch of mixed lengths is bit-identical to each waveform analysed alone, and to the host entry.
  3. wrnn_score_wav_many is bit-identical to wrnn_score_many fed the device's own mel and targets, on the persistent,
     SIMT and stream engines (MoL) and the persistent engine (RAW, mu-law and linear), with and without peak_norm and
     with a recording whose peak exceeds 1.
  4. The shipped checkpoint finds its own vocoded speech more likely than noise of the same RMS.
Run on a GPU: pytest -m gpu -s tests/test_gpu_mel.py"""
import numpy as np
import pytest
import torch

import helpers
import mel_oracle as MO
from test_mel_abi import CONFIGS, MEL_TOL
from wavernn_b200 import cabi

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def speech():
    return helpers.load_golden("trained_tacotron.npz")["wav"].astype(np.float32)


def signals(n_fft):
    s = dict(MO.signals(), speech=speech())
    s["minimum"] = MO.signals()["noise_full"][:n_fft // 2 + 1].copy()
    rs = np.random.RandomState(7)
    ten = np.tile(speech(), 22050 * 600 // speech().size + 1)[:22050 * 600]
    s["ten_minutes"] = (ten + 0.01 * rs.randn(ten.size)).astype(np.float32)
    return s


def mels_device(an, ys):
    """wrnn_melspectrogram_many on device copies of ys (one batch); returns the host mels."""
    dy = [torch.as_tensor(y, device=DEV) for y in ys]
    dm = [torch.full((an.cfg.n_mels, an.frames(y.size)), float("nan"), device=DEV) for y in ys]
    an.melspectrogram_many(ys=[y.data_ptr() for y in dy], ns=[y.size for y in ys], mels=[m.data_ptr() for m in dm],
                           stream=torch.cuda.current_stream(DEV).cuda_stream)
    torch.cuda.synchronize(DEV)
    return [m.cpu().numpy() for m in dm]


@pytest.mark.parametrize("name", list(CONFIGS))
def test_kernel_against_oracle(name):
    cfg = CONFIGS[name]
    an = cabi.MelAnalysis(**cfg)
    try:
        sigs = signals(an.cfg.n_fft)
        got = mels_device(an, list(sigs.values()))
        worst = {}
        for (k, y), g in zip(sigs.items(), got):
            ref = MO.melspectrogram(y, **cfg)
            assert g.shape == ref.shape and g.dtype == np.float32, k
            worst[k] = float(np.abs(g - ref).max())
            if k == "silence_click":
                silent = ref.max(axis=0) == 0
                assert silent.sum() > 10 and (g[:, silent] == 0).all()
        print(f"{name}: max |kernel - oracle| " + ", ".join(f"{k} {v:.2e}" for k, v in worst.items()))
        assert max(worst.values()) <= MEL_TOL, worst
    finally:
        an.close()


def test_batch_equals_single():
    an = cabi.MelAnalysis()
    try:
        rs = np.random.RandomState(3)
        ys = [(0.3 * rs.randn(n)).astype(np.float32) for n in (1025, 44825, 2199, 2200, 100000, 5001)]
        batch = mels_device(an, ys)
        for i, y in enumerate(ys):
            assert np.array_equal(mels_device(an, [y])[0], batch[i]), i
        host = an.melspectrogram_many_host(ys)
        assert all(np.array_equal(a, b) for a, b in zip(host, batch))
        perm = [5, 2, 0, 4, 1, 3]
        pb = mels_device(an, [ys[i] for i in perm])
        assert all(np.array_equal(pb[k], batch[i]) for k, i in enumerate(perm))
    finally:
        an.close()


def recordings():
    s = speech()[:9000]
    rs = np.random.RandomState(11)
    return [s, (3.0 * s).astype(np.float32), np.clip(0.4 * rs.randn(6000), -1, 1).astype(np.float32)]


def composed(eng, an, ys, peak_norm, mu_law):
    """wrnn_score_many fed the device's normalised recordings' mels (wrnn_melspectrogram_many) and targets
    (wrnn_debug_score_wav_targets); returns (nll list, target list)."""
    lib, s = cabi.load(), torch.cuda.current_stream(DEV).cuda_stream
    mode, nc = (0, 30) if eng.mode == "MOL" else (1, eng.n_classes)
    nlls, xs = [], []
    for y in ys:
        dy = torch.as_tensor(y, device=DEV)
        yn, x, peak = torch.empty_like(dy), torch.empty_like(dy), torch.empty(1, device=DEV)
        assert lib.wrnn_debug_score_wav_targets(dy.data_ptr(), y.size, mode, nc, int(peak_norm), int(mu_law), yn.data_ptr(),
                                                x.data_ptr(), peak.data_ptr(), s) == 0
        mel = torch.empty((80, an.frames(y.size)), device=DEV)
        an.melspectrogram_many(ys=[yn.data_ptr()], ns=[y.size], mels=[mel.data_ptr()], stream=s)
        nll = torch.full((y.size,), float("nan"), device=DEV)
        eng.score_many(mels=[mel.data_ptr()], Ts=[mel.shape[1]], xs=[x.data_ptr()], ns=[y.size], nlls=[nll.data_ptr()], stream=s)
        torch.cuda.synchronize(DEV)
        eng.check()
        nlls.append(nll.cpu().numpy())
        xs.append(x.cpu().numpy())
    return nlls, xs


def score_wav_device(eng, an, ys, peak_norm, mu_law):
    dy = [torch.as_tensor(y, device=DEV) for y in ys]
    dn = [torch.full((y.size,), float("nan"), device=DEV) for y in ys]
    eng.score_wav_many(an, ys=[y.data_ptr() for y in dy], ns=[y.size for y in ys], nlls=[o.data_ptr() for o in dn],
                       peak_norm=peak_norm, mu_law=mu_law, stream=torch.cuda.current_stream(DEV).cuda_stream)
    torch.cuda.synchronize(DEV)
    eng.check()
    return [o.cpu().numpy() for o in dn]


COMPOSITION = [("MOL", "tcgen05", "fp16", False), ("MOL", "simt", "fp32", False), ("MOL", "stream", "fp16", False),
               ("RAW", "tcgen05", "fp16", True), ("RAW", "tcgen05", "bf16", False)]


@pytest.mark.parametrize("head,engine,precision,mu_law", COMPOSITION,
                         ids=[f"{h}-{e}-{p}-{'mu' if u else 'lin'}" for h, e, p, u in COMPOSITION])
def test_score_wav_is_score_many_of_its_mel_and_targets(head, engine, precision, mu_law):
    m = helpers.make_model(0, head)
    eng = cabi.Engine(m.hot_state(), n_classes=m.n_classes, mode=head, precision=precision, engine=engine)
    an = cabi.MelAnalysis()
    try:
        eng.attach_upsampler(m.state_dict())
        ys = recordings()
        bits = 16 if head == "MOL" else int(np.log2(m.n_classes))
        for peak_norm in (False, True):
            batch = score_wav_device(eng, an, ys, peak_norm, mu_law)
            ref, xs = composed(eng, an, ys, peak_norm, mu_law)
            for i, y in enumerate(ys):
                assert np.isfinite(batch[i]).all(), i
                assert np.array_equal(batch[i], ref[i]), (eng.name, peak_norm, i)
                want = MO.targets(MO.normalise(y, peak_norm), head, bits, mu_law)
                moved = int((xs[i] != want).sum())
                # MoL and linear labels are exact; a mu-law code may move by one where numpy's float32 log and the
                # library's rounded double log straddle a code boundary
                assert moved == 0 if not mu_law else moved <= 2, (i, moved)
            host = eng.score_wav_many_host(an, ys, peak_norm=peak_norm, mu_law=mu_law)
            assert all(np.array_equal(a, b) for a, b in zip(host, batch)), (eng.name, "host")
        print(f"score_wav_many {head} [{eng.name}] mu_law={mu_law}: bit-identical to score_many of its mel and targets; "
              f"mean nll {[float(b.mean()) for b in batch]}")
        with pytest.raises(cabi.EngineError, match="hop_length"):
            other = cabi.MelAnalysis(hop_length=256)
            try:
                eng.score_wav_many_host(other, ys[:1])
            finally:
                other.close()
    finally:
        an.close()
        eng.close()


def test_checkpoint_prefers_its_own_speech():
    model = helpers.make_model(0, "MOL", "cpu")
    model.load_state_dict(helpers.pretrained_state_dict(), strict=False)
    eng = cabi.Engine(model.hot_state(), n_classes=30, mode="MOL", precision="fp16", engine="tcgen05")
    an = cabi.MelAnalysis()
    try:
        eng.attach_upsampler(model.state_dict())
        y = speech()
        mel = an.melspectrogram_many_host([y])[0]
        g = helpers.load_golden("trained_tacotron.npz")
        taco = helpers.tacotron_mels()[int(g["sentence"])]
        n = min(taco.shape[1], mel.shape[1])
        print(f"analysed mel {mel.shape} vs Tacotron mel {taco.shape}: mean |diff| {np.abs(mel[:, :n] - taco[:, :n]).mean():.4f}")
        rs = np.random.RandomState(0)
        noise = (rs.randn(y.size) * np.sqrt(np.mean(y.astype(np.float64) ** 2))).astype(np.float32)
        s_nll, n_nll = eng.score_wav_many_host(an, [y, noise])
        print(f"mean nll: own speech {s_nll.mean():.4f}, noise at the same RMS {n_nll.mean():.4f}")
        assert np.isfinite(s_nll).all() and s_nll.mean() < n_nll.mean()
    finally:
        an.close()
        eng.close()
