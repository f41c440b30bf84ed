"""The mel analysis and scoring from audio, checked without a device: the oracle (tests/mel_oracle.py) against an
independent implementation (tests/golden/mel_pins.npz), the negative control of the kernel's tolerance, the tables
wrnn_mel_create builds on the host, the kernel's per-frame code run on the host, the ctypes mirrors, the frame table
and the refusals of every new entry point, and the quantiser of wrnn_score_wav_many."""
import ctypes
import subprocess

import numpy as np
import pytest

import helpers
import mel_oracle as MO
from wavernn_b200 import cabi

ROOT = helpers.GOLDEN.parent.parent
# The kernel's tolerance against the oracle, in normalized units, for every signal and configuration.  Each output is
# the float32 rounding of a float64 quantity that the kernel and the oracle both compute to about 1e-12 (rounding each
# bin to complex64, the one rounding inside, moves a band's dB value by far less).  Outputs lie in [0, 1], where a
# float32 step is at most 2^-24, so two such roundings differ by at most one step plus the float64 gap: 2^-23 leaves a
# margin of one step.  tests/test_mel_edges.py holds it on every configuration of its grid; log10 in float32 misses it.
MEL_TOL = 2.0 ** -23
FAKE = 0x1000                      # the plan hooks only test pointers against NULL
CONFIGS = {"default": {}, "1024-1024-256": dict(n_fft=1024, win_length=1024, hop_length=256), "n_fft4096": dict(n_fft=4096),
           "n_mels128": dict(n_mels=128), "fmin0": dict(fmin=0.0)}


@pytest.fixture(scope="module")
def lib():
    if not cabi.is_built():
        import __graft_entry__ as g
        g.build()
    return cabi.load()


def speech():
    return helpers.load_golden("trained_tacotron.npz")["wav"].astype(np.float32)


def test_oracle_matches_independent_fixture():
    """torch.stft + torchaudio's Slaney filterbank (float64) against the oracle: measured 1.07e-6 on the mel and 4.3e-6
    relative on the filterbank (torchaudio's is built in float32)."""
    p = helpers.load_golden("mel_pins.npz")
    d_mel = np.abs(MO.melspectrogram(speech()) - p["mel"]).max()
    d_fb = np.abs(MO.mel_basis(**MO.DEFAULT) - p["fbank"]).max() / p["fbank"].max()
    print(f"oracle vs torch/torchaudio: mel {d_mel:.3e}, filterbank {d_fb:.3e} relative")
    assert d_mel <= 4e-6 and d_fb <= 2e-5
    assert p["mel"].shape == (80, 1 + speech().size // 275) == (80, 164)


def test_float32_fft_fails_the_tolerance():
    """Negative control: the single-precision transform on the 0.9-amplitude 440 Hz tone misses MEL_TOL by far, so the
    tolerance tells the two precisions apart."""
    y = MO.signals()["tone440"]
    d = np.abs(MO.melspectrogram(y) - MO.melspectrogram(y, fft_dtype=np.float32)).max()
    print(f"float32 FFT vs float64 FFT on the tone: {d:.3e} (tolerance {MEL_TOL})")
    assert d > 10 * MEL_TOL


@pytest.mark.parametrize("name", list(CONFIGS))
def test_host_tables(lib, name):
    c = dict(MO.DEFAULT, **CONFIGS[name])
    cfg = cabi.mel_cfg(**c)
    nb = c["n_fft"] // 2 + 1
    win, basis = np.zeros(c["n_fft"]), np.zeros((c["n_mels"], nb))
    bands = np.zeros((c["n_mels"], 2), dtype=np.int32)
    assert lib.wrnn_debug_mel_tables(ctypes.byref(cfg), win.ctypes.data, basis.ctypes.data, bands.ctypes.data) == 0
    np.testing.assert_allclose(win, MO.window(**c), rtol=0, atol=1e-15)
    ref = MO.mel_basis(**c)
    np.testing.assert_allclose(basis, ref, rtol=1e-12, atol=1e-15)
    for m in range(c["n_mels"]):
        nz = np.flatnonzero(basis[m] > 0)
        assert np.array_equal(nz, np.flatnonzero(ref[m] > 0)), m
        lo, cnt = bands[m]
        assert cnt == nz.size and (cnt == 0 or (lo == nz[0] and nz[-1] == lo + cnt - 1)), m


def host_frames(lib, y, **cfg):
    c = dict(MO.DEFAULT, **cfg)
    y = np.ascontiguousarray(y, dtype=np.float32)
    out = np.full((c["n_mels"], 1 + y.size // c["hop_length"]), np.nan, dtype=np.float32)
    rc = lib.wrnn_debug_mel_frames(ctypes.byref(cabi.mel_cfg(**c)), y.ctypes.data, y.size, out.ctypes.data)
    assert rc == 0, lib.wrnn_last_error().decode()
    return out


@pytest.mark.parametrize("name", list(CONFIGS))
def test_kernel_code_on_the_host(lib, name):
    """The kernel's per-frame functions run on the host against the oracle, held to the GPU tolerance."""
    cfg = CONFIGS[name]
    sigs = dict(MO.signals(seconds=0.5), speech=speech())
    worst = 0.0
    for k, y in sigs.items():
        got, ref = host_frames(lib, y, **cfg), MO.melspectrogram(y, **cfg)
        worst = max(worst, float(np.abs(got - ref).max()))
        if k == "silence_click":
            assert (got[:, ref.max(axis=0) == 0] == 0).all()
    print(f"{name}: host run of the kernel code vs oracle {worst:.3e}")
    assert worst <= MEL_TOL


def test_struct_layouts_match_header(tmp_path):
    structs = {"wrnn_mel_cfg": (cabi.WrnnMelCfg, 28), "wrnn_mel_utt": (cabi.WrnnMelUtt, 24),
               "wrnn_score_wav_utt": (cabi.WrnnScoreWavUtt, 24)}
    lines = ["#include <stddef.h>", "#include <stdio.h>", '#include "wavernn_b200.h"', "int main(void) {"]
    for s, (py, _) in structs.items():
        lines.append(f'  printf("{s} size %zu\\n", sizeof({s}));')
        lines += [f'  printf("{s} {f} %zu\\n", offsetof({s}, {f}));' for f, _ in py._fields_]
    lines += ["  return 0;", "}"]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines) + "\n")
    exe = tmp_path / "layout"
    subprocess.run(["cc", "-std=c99", "-I", str(ROOT / "include"), "-o", str(exe), str(src)], check=True)
    got = {" ".join(l.split()[:2]): int(l.split()[2]) for l in
           subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines()}
    for s, (py, size) in structs.items():
        assert got[f"{s} size"] == ctypes.sizeof(py) == size, s
        for f, _ in py._fields_:
            assert got[f"{s} {f}"] == getattr(py, f).offset, (s, f)


CFG_REFUSALS = [
    (dict(sample_rate=0), "sample_rate"), (dict(n_fft=128), "n_fft"), (dict(n_fft=8192), "n_fft"), (dict(n_fft=2000), "n_fft"),
    (dict(hop_length=0), "hop_length"), (dict(win_length=0), "win_length"), (dict(win_length=2049), "win_length"),
    (dict(n_mels=0), "n_mels"), (dict(n_mels=129), "n_mels"), (dict(fmin=-1.0), "fmin"), (dict(fmin=11025.0), "fmin"),
    (dict(fmin=float("nan")), "fmin"), (dict(min_level_db=0.0), "min_level_db"), (dict(min_level_db=float("-inf")), "min_level_db"),
]


@pytest.mark.parametrize("kw,msg", CFG_REFUSALS, ids=[f"{m}-{i}" for i, (_, m) in enumerate(CFG_REFUSALS)])
def test_create_refuses_before_the_device(lib, kw, msg):
    m = ctypes.c_void_p()
    assert lib.wrnn_mel_create(ctypes.byref(m), ctypes.byref(cabi.mel_cfg(**kw)), 0) == cabi.WRNN_E_INVALID
    assert msg in lib.wrnn_last_error().decode() and not m.value
    assert lib.wrnn_debug_mel_tables(ctypes.byref(cabi.mel_cfg(**kw)), None, None, None) == cabi.WRNN_E_INVALID


def mel_plan(lib, ns, null=None, **cfg):
    items = [(FAKE, n, FAKE) for n in ns]
    if null is not None:
        i, field = null
        items[i] = (0 if field == "y" else FAKE, ns[i], 0 if field == "mel" else FAKE)
    arr, n = cabi.utt_array(cabi.WrnnMelUtt, items)
    f0 = np.zeros(max(n, 1) + 1, dtype=np.int64)
    rc = lib.wrnn_debug_mel_plan(ctypes.byref(cabi.mel_cfg(**cfg)), arr, n, f0.ctypes.data)
    return rc, lib.wrnn_last_error().decode() if rc else "", f0


def test_frame_table(lib):
    hop = 275
    ns = [8 * hop - 1, 8 * hop, 1025, 44825, 8 * hop + 1]
    rc, msg, f0 = mel_plan(lib, ns)
    assert rc == 0, msg
    T = np.diff(f0)
    assert list(T) == [1 + n // hop for n in ns] == [8, 9, 4, 164, 9]
    assert f0[0] == 0 and f0[-1] == sum(T)
    for n_fft, hop, win in ((1024, 256, 1024), (4096, 275, 1100)):
        ns = [8 * hop - 1, 8 * hop, n_fft // 2 + 1]
        rc, msg, f0 = mel_plan(lib, ns, n_fft=n_fft, hop_length=hop, win_length=win)
        assert rc == 0 and list(np.diff(f0)) == [1 + n // hop for n in ns], msg


MEL_REFUSALS = [
    (dict(ns=()), "non-null utterance array"),
    (dict(ns=(5000, 1024)), "utterance 1: n must be > n_fft / 2 = 1024"),
    (dict(ns=(1025, 5000), n_fft=4096), "utterance 0: n must be > n_fft / 2 = 2048"),
    (dict(ns=(5000, 5000), null=(1, "y")), "utterance 1: y and mel are required"),
    (dict(ns=(5000,), null=(0, "mel")), "utterance 0: y and mel are required"),
    (dict(ns=(2 ** 40, 2 ** 40), hop_length=1), "2^31 frames"),
]


@pytest.mark.parametrize("kw,msg", MEL_REFUSALS, ids=[m.split(":")[0] + f"-{i}" for i, (_, m) in enumerate(MEL_REFUSALS)])
def test_melspectrogram_refusals(lib, kw, msg):
    rc, got, _ = mel_plan(lib, **kw)
    assert rc == cabi.WRNN_E_INVALID and msg in got, got


def test_null_analysis_object_is_refused(lib):
    arr, n = cabi.utt_array(cabi.WrnnMelUtt, [(FAKE, 5000, FAKE)])
    assert lib.wrnn_melspectrogram_many(None, arr, n, None) == cabi.WRNN_E_INVALID
    assert lib.wrnn_melspectrogram_many_host(None, arr, n) == cabi.WRNN_E_INVALID
    assert "null analysis object" in lib.wrnn_last_error().decode()
    sarr, n = cabi.utt_array(cabi.WrnnScoreWavUtt, [(FAKE, 5000, FAKE)])
    assert lib.wrnn_score_wav_many(None, None, sarr, n, 0, 0, None) == cabi.WRNN_E_INVALID
    assert lib.wrnn_score_wav_many_host(None, None, sarr, n, 0, 0) == cabi.WRNN_E_INVALID
    assert "null handle" in lib.wrnn_last_error().decode()


def wav_plan(lib, ns, feat=80, hop=275, null=None, **cfg):
    items = [(FAKE, n, FAKE) for n in ns]
    if null is not None:
        i, field = null
        items[i] = (0 if field == "y" else FAKE, ns[i], 0 if field == "nll" else FAKE)
    arr, n = cabi.utt_array(cabi.WrnnScoreWavUtt, items)
    T = np.zeros(max(n, 1), dtype=np.int64)
    rc = lib.wrnn_debug_score_wav_plan(feat, hop, ctypes.byref(cabi.mel_cfg(**cfg)), arr, n, T.ctypes.data)
    return rc, lib.wrnn_last_error().decode() if rc else "", T


def test_score_wav_job(lib):
    """Each recording becomes a wrnn_score_many utterance of T = 1 + n // hop frames, so that every sample is scored."""
    ns = [8 * 275 - 1, 8 * 275, 1025, 44825]
    rc, msg, T = wav_plan(lib, ns)
    assert rc == 0, msg
    assert list(T) == [1 + n // 275 for n in ns] and all(t * 275 >= n for t, n in zip(T, ns))


WAV_REFUSALS = [
    (dict(ns=(5000,), feat=81), "n_mels = 80 bands, the model takes feat_dims = 81"),
    (dict(ns=(5000,), hop=256), "hop_length 275, the attached upsampler hop_length 256"),
    (dict(ns=()), "1 to 65535 utterances"),
    (dict(ns=(5000,) * 65536), "1 to 65535 utterances"),
    (dict(ns=(5000, 1024)), "utterance 1: n must be > n_fft / 2 = 1024"),
    (dict(ns=(5000, 5000), null=(1, "y")), "utterance 1: y and nll are required"),
    (dict(ns=(5000,), null=(0, "nll")), "utterance 0: y and nll are required"),
    (dict(ns=(2 ** 31 - 4 * 275,) * 2), "2^31"),
]


@pytest.mark.parametrize("kw,msg", WAV_REFUSALS, ids=[f"{i}" for i in range(len(WAV_REFUSALS))])
def test_score_wav_refusals(lib, kw, msg):
    rc, got, _ = wav_plan(lib, **kw)
    assert rc == cabi.WRNN_E_INVALID and msg in got, got


QUANT = [("MOL", 16, False), ("RAW", 9, True), ("RAW", 9, False), ("RAW", 10, True)]


@pytest.mark.parametrize("mode,bits,mu_law", QUANT, ids=[f"{m}-{b}-{'mu' if u else 'lin'}" for m, b, u in QUANT])
def test_quantiser(lib, mode, bits, mu_law):
    """The float32 restatement round-trips the label grid -- every label is reached, its target is label_2_float of it,
    and the scoring kernels read the label back from the target (rint((x + 1)(2^bits - 1) / 2)) -- and the library's
    quantiser (run on the host) equals it."""
    top = 2 ** (16 if mode == "MOL" else bits) - 1
    grid = np.arange(top + 1)
    l2f = lambda L: (np.float32(2) * L.astype(np.float32)) / np.float32(top) - np.float32(1)
    probe = np.linspace(-1, 1, 4 * (top + 1), dtype=np.float32)
    if mu_law:   # the decoded code values (utils/dsp.py decode_mu_law) encode back to their codes
        ys = l2f(grid)
        ys = (np.sign(ys) / top * ((1 + top) ** np.abs(ys.astype(np.float64)) - 1)).astype(np.float32)
        assert np.array_equal(MO.labels(ys, mode, bits, True), grid)
        probe = np.concatenate([probe, ys])
    L = MO.labels(probe, mode, bits, mu_law)
    assert np.array_equal(np.unique(L), grid)
    x = MO.targets(probe, mode, bits, mu_law)
    assert x.dtype == np.float32 and np.array_equal(x, l2f(L))
    assert np.array_equal(np.rint((x.astype(np.float64) + 1) * top / 2).astype(np.int64), L)
    rs = np.random.RandomState(bits)
    y = np.concatenate([probe, l2f(grid), np.clip(rs.randn(20000) * 0.3, -1, 1), [-1, 1, 0, -0.0, 1e-9, -1e-9]]).astype(np.float32)
    got = np.empty_like(y)
    assert lib.wrnn_debug_wav_targets(y.ctypes.data, y.size, 0 if mode == "MOL" else 1, 30 if mode == "MOL" else 2 ** bits,
                                      int(mu_law), got.ctypes.data) == 0
    assert np.array_equal(got, MO.targets(y, mode, bits, mu_law))


def test_normalise():
    y = np.array([0.5, -2.0, 1.0], dtype=np.float32)
    assert np.array_equal(MO.normalise(y, False), y / np.float32(2.0))
    y = np.array([0.5, -0.25], dtype=np.float32)
    assert np.array_equal(MO.normalise(y, False), y) and np.array_equal(MO.normalise(y, True), y / np.float32(0.5))
