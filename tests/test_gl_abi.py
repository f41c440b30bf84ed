"""Griffin-Lim (wrnn_griffinlim_many) checked without a device: the oracle (tests/gl_oracle.py) against torch.stft,
torch.istft and torchaudio's griffinlim, the library's NNLS against librosa 0.7's on the 16 Tacotron mels, the kernels'
per-frame code run on the host (wrnn_debug_griffinlim) against the oracle at every configuration of
test_mel_abi.CONFIGS and more, the ctypes mirror, the frame table and the refusals."""
import ctypes
import subprocess

import numpy as np
import pytest
import torch
import torchaudio

import gl_oracle as G
import helpers
import mel_oracle as MO
from test_mel_abi import CONFIGS, FAKE, ROOT
from wavernn_b200 import cabi

# n_iter 0 and 1: the output is linear in S (n_iter 0) or one phase update away from it, and the host run of the kernel
# code differs from the oracle only in the last bits of the float64 transforms: measured 0 and 1 float32 step of the
# peak on the Tacotron mels; 4 steps leaves margin.
ULPS_EARLY = 4
# n_iter 32: momentum 0.99 amplifies last-bit differences chaotically.  Calibration on the oracle over the 16 Tacotron
# mels (peak about 0.2): noise of 1e-15 of each frame's peak added to both FFTs moves the output by up to 7.8e-5; one
# float32 step added to 0.1 % of the bins of S (what a differently rounded float64 solve does) by up to 3.4e-4 (two sets
# of seeds).  Implementations that differ only in such bits were measured at up to 1.2e-3 (the host run of the kernel
# code, seeds 0-15) and 3.5e-4 (the device): the tail is heavy, so the tolerance is 3e-3, 1.5 % of the peak -- still far
# below what any change of algorithm gives (another NNLS solver or another seed: about 40 % relative L2).
GL32_TOL = 3e-3
# the configurations of the host-run check: test_mel_abi's, a one-sample window, and n_fft = 256 with 128 bands (many of
# them empty or sharing one bin, so the start solve drops bands)
GL_CONFIGS = dict(CONFIGS, win1=dict(win_length=1), fft256_mels128=dict(n_fft=256, win_length=255, hop_length=200, n_mels=128))


@pytest.fixture(scope="module")
def lib():
    if not cabi.is_built():
        import __graft_entry__ as g
        g.build()
    return cabi.load()


def speech():
    return helpers.load_golden("trained_tacotron.npz")["wav"].astype(np.float32)


def test_oracle_matches_torch():
    """The oracle's istft / stft pair (float32, as librosa 0.7 runs it) against torch.istft / torch.stft in float64,
    and its Griffin-Lim from all-ones phases in float64 against torchaudio.functional.griffinlim (whose momentum
    argument is librosa's momentum / (1 + momentum)).  Measured: istft 1.0e-8 of a 0.07 peak (1.3 float32 steps), stft
    2.4e-7 of a 6.8 peak (the complex64 rounding), Griffin-Lim 1.4e-14 (0 iterations) and 3.7e-10 (1 iteration) relative to the peak.  From the
    second iteration on, bins whose magnitude sits at the transforms' rounding noise take their phase from that noise,
    so only the first two stages are compared."""
    c = dict(MO.DEFAULT)
    N, hop, W = c["n_fft"], c["hop_length"], c["win_length"]
    win = torch.hann_window(W, periodic=True, dtype=torch.float64)
    for mel in (helpers.tacotron_mels()[15], helpers.tacotron_mels()[9]):
        S = G.mel_to_stft(mel, **c)
        T, L = S.shape[1], hop * (S.shape[1] - 1)
        X = (S * G.phases(1, T, S.shape[0])).astype(np.complex64)
        y = G.istft(X, **c)
        ref = torch.istft(torch.from_numpy(X.astype(np.complex128)), N, hop, W, win, center=True, length=L).numpy()
        assert y.dtype == np.float32 and y.shape == (L,)
        assert np.abs(y - ref).max() <= 4 * np.spacing(np.float32(np.abs(ref).max()))
        R = G.stft(y, **c)
        Rt = torch.stft(torch.from_numpy(y.astype(np.float64)), N, hop, W, win, center=True, pad_mode="reflect",
                        return_complex=True).numpy()
        assert R.dtype == np.complex64 and R.shape == S.shape
        assert np.abs(R - Rt).max() <= 1e-6 * np.abs(Rt).max()
        for n_iter, tol in ((0, 1e-12), (1, 1e-8)):
            got = G.griffinlim(S, np.ones(S.shape), n_iter, dtype=np.float64, **c)
            want = torchaudio.functional.griffinlim(torch.from_numpy(S.astype(np.float64)), win, N, hop, W, 1.0, n_iter,
                                                    G.MOMENTUM / (1 + G.MOMENTUM), L, False).numpy()
            d = np.abs(got - want).max() / np.abs(want).max()
            print(f"T={T} n_iter={n_iter}: oracle vs torchaudio {d:.2e} of the peak")
            assert d <= tol


def test_fista_against_lbfgs_on_tacotron_mels():
    """On all 16 Tacotron mels the library's solve is non-negative, leaves a relative residual no larger than librosa
    0.7's L-BFGS-B on every frame, and lands within a few percent of its solution (the minimiser is not unique)."""
    c = dict(MO.DEFAULT)
    A = G.fb32(**c)
    dist = []
    for i, mel in enumerate(helpers.tacotron_mels()):
        B = G.amplitudes(mel, **c)
        xf, xl = G.nnls_fista(A, B, dtype=np.float64), G.nnls_lbfgs(A, B, dtype=np.float64)
        rf, rl = G.rel_residual(A, B, xf), G.rel_residual(A, B, xl)
        assert (xf >= 0).all(), i
        assert (rf <= np.maximum(rl, 1e-30)).all(), (i, np.flatnonzero(rf > rl)[:5], rf.max(), rl.max())
        dist.append(np.linalg.norm(xf - xl) / np.linalg.norm(xl))
        print(f"mel_{i:02d}: residual FISTA median {np.median(rf):.1e} max {rf.max():.1e}, L-BFGS-B median "
              f"{np.median(rl):.1e} max {rl.max():.1e}, distance {dist[-1]:.2%}")
    assert max(dist) <= 0.05


def host_gl(lib, mel, seed, n_iter, **cfg):
    """wrnn_debug_griffinlim: the kernels' code run on the host -> (wav, S [n_bins, T])."""
    c = dict(MO.DEFAULT, **cfg)
    mel = np.ascontiguousarray(mel, dtype=np.float32)
    T = mel.shape[1]
    wav = np.full(c["hop_length"] * (T - 1), np.nan, dtype=np.float32)
    S = np.full((T, c["n_fft"] // 2 + 1), np.nan, dtype=np.float32)
    rc = lib.wrnn_debug_griffinlim(ctypes.byref(cabi.mel_cfg(**c)), mel.ctypes.data, T, seed, n_iter, wav.ctypes.data,
                                   S.ctypes.data)
    assert rc == 0, lib.wrnn_last_error().decode()
    return wav, S.T


def config_mel(name):
    """A mel of the configuration: the oracle's analysis of the speech fixture, cut to about 40 frames."""
    c = dict(MO.DEFAULT, **GL_CONFIGS[name])
    n = max(40 * c["hop_length"], c["n_fft"])
    return MO.melspectrogram(speech()[:n], **c), c


@pytest.mark.parametrize("name", list(GL_CONFIGS))
def test_kernel_code_on_the_host_early_iterations(lib, name):
    mel, c = config_mel(name)
    S_ref = G.mel_to_stft(mel, **c)
    for n_iter in (0, 1, 2):
        got, S = host_gl(lib, mel, 7, n_iter, **c)
        if n_iter == 0:
            dS = np.abs(S - S_ref).max() / max(S_ref.max(), 1e-30)
            print(f"{name}: S vs oracle {dS:.2e} of the peak")
            assert dS <= 1e-5
        ref = G.griffinlim(S_ref, G.phases(7, S_ref.shape[1], S_ref.shape[0]), n_iter, **c)
        steps = np.abs(got - ref).max() / np.spacing(np.abs(ref).max())
        print(f"{name}: n_iter={n_iter}: {steps:.1f} float32 steps of the peak")
        assert got.shape == ref.shape and steps <= (ULPS_EARLY if n_iter < 2 else 64)


def test_kernel_code_on_the_host_32_iterations(lib):
    worst = 0.0
    for i, mel in enumerate(helpers.tacotron_mels()):
        got, S = host_gl(lib, mel, i, 32)
        ref = G.griffinlim(S, G.phases(i, S.shape[1], S.shape[0]), 32)
        worst = max(worst, float(np.abs(got - ref).max()))
    print(f"32 iterations on the 16 Tacotron mels: host run vs oracle {worst:.2e} (tolerance {GL32_TOL})")
    assert worst <= GL32_TOL


def test_phases_are_keyed_by_seed_frame_and_bin(lib):
    """The host run's n_iter = 0 output is the istft of S times the oracle's Philox phases; other seeds differ."""
    mel = helpers.tacotron_mels()[15][:, :30]
    a, S = host_gl(lib, mel, 3, 0)
    b, _ = host_gl(lib, mel, 3 + (1 << 40), 0)
    assert np.array_equal(a, G.istft(S * G.phases(3, 30, S.shape[0]), **MO.DEFAULT))
    assert not np.array_equal(a, b)
    ph = G.phases(3, 30, 1025)
    assert ph.dtype == np.complex64 and np.allclose(np.abs(ph), 1, atol=1e-6)


def test_struct_layout_matches_header(tmp_path):
    py = cabi.WrnnGlUtt
    lines = ["#include <stddef.h>", "#include <stdio.h>", '#include "wavernn_b200.h"', "int main(void) {",
             '  printf("size %zu\\n", sizeof(wrnn_gl_utt));']
    lines += [f'  printf("{f} %zu\\n", offsetof(wrnn_gl_utt, {f}));' for f, _ in py._fields_]
    lines += ["  return 0;", "}"]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines) + "\n")
    exe = tmp_path / "layout"
    subprocess.run(["cc", "-std=c99", "-I", str(ROOT / "include"), "-o", str(exe), str(src)], check=True)
    got = dict((l.split()[0], int(l.split()[1])) for l in
               subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    assert got["size"] == ctypes.sizeof(py) == 32
    for f, _ in py._fields_:
        assert got[f] == getattr(py, f).offset, f


def gl_plan(lib, Ts, n_iter=32, null=None, **cfg):
    items = [(FAKE, T, 0, FAKE) for T in Ts]
    if null is not None:
        i, field = null
        items[i] = (0 if field == "mel" else FAKE, Ts[i], 0, 0 if field == "wav" else FAKE)
    arr, n = cabi.utt_array(cabi.WrnnGlUtt, items)
    f0 = np.zeros(max(n, 1) + 1, dtype=np.int64)
    rc = lib.wrnn_debug_griffinlim_plan(ctypes.byref(cabi.mel_cfg(**cfg)), arr, n, n_iter, f0.ctypes.data)
    return rc, lib.wrnn_last_error().decode() if rc else "", f0


def test_frame_table(lib):
    Ts = [5, 318, 6, 1000, 98]   # T = 5 is the shortest at the defaults: 275 * 4 > 1024
    rc, msg, f0 = gl_plan(lib, Ts)
    assert rc == 0, msg
    assert list(np.diff(f0)) == Ts and f0[0] == 0
    for n_iter in (0, 1, 1000):
        assert gl_plan(lib, Ts, n_iter)[0] == 0
    rc, msg, f0 = gl_plan(lib, [3, 4], n_fft=1024, hop_length=256, win_length=1024)   # 256 * 2 = 512 is not > 512
    assert rc == cabi.WRNN_E_INVALID and "utterance 0" in msg
    rc, msg, f0 = gl_plan(lib, [4, 3], n_fft=1024, hop_length=256, win_length=1024)
    assert rc == cabi.WRNN_E_INVALID and "utterance 1" in msg


GL_REFUSALS = [
    (dict(Ts=()), "non-null utterance array"),
    (dict(Ts=(300, 4)), "utterance 1: hop_length * (T - 1) must be > n_fft / 2 = 1024"),
    (dict(Ts=(1, 300)), "utterance 0: hop_length * (T - 1) must be > n_fft / 2 = 1024"),
    (dict(Ts=(0,)), "utterance 0: hop_length * (T - 1)"),
    (dict(Ts=(-5,)), "utterance 0: hop_length * (T - 1)"),
    (dict(Ts=(300, 6), n_fft=4096), "utterance 1: hop_length * (T - 1) must be > n_fft / 2 = 2048"),
    (dict(Ts=(300, 300), null=(1, "mel")), "utterance 1: mel and wav are required"),
    (dict(Ts=(300,), null=(0, "wav")), "utterance 0: mel and wav are required"),
    (dict(Ts=(2 ** 30, 2 ** 30)), "2^31 frames"),
    (dict(Ts=(2 ** 62,)), "2^31 frames"),
    (dict(Ts=(300,), n_iter=-1), "n_iter must be >= 0"),
]


@pytest.mark.parametrize("kw,msg", GL_REFUSALS, ids=[f"{i}" for i in range(len(GL_REFUSALS))])
def test_griffinlim_refusals(lib, kw, msg):
    rc, got, _ = gl_plan(lib, **kw)
    assert rc == cabi.WRNN_E_INVALID and msg in got, got


def test_null_analysis_object_is_refused(lib):
    arr, n = cabi.utt_array(cabi.WrnnGlUtt, [(FAKE, 300, 0, FAKE)])
    assert lib.wrnn_griffinlim_many(None, arr, n, 32, None) == cabi.WRNN_E_INVALID
    assert lib.wrnn_griffinlim_many_host(None, arr, n, 32) == cabi.WRNN_E_INVALID
    assert "null analysis object" in lib.wrnn_last_error().decode()


def test_exports():
    assert {"wrnn_griffinlim_many", "wrnn_griffinlim_many_host"} <= set(cabi.EXPORTS)
