"""The resampling step of load_wav without a GPU: the library's filter table against the numpy/scipy design, its host
hook (the kernel's per-output function run on the CPU) bit for bit against tests/resample_oracle.py, the oracle against
analytic tones and torchaudio, and the C surface (length, struct layout, refusals)."""
import ctypes as C

import numpy as np
import pytest

import resample_oracle as R
from wavernn_b200 import cabi

RATES = (44100, 48000, 16000, 8000, 24000, 22051, 22050)
SR = 22050


@pytest.fixture(scope="module")
def lib():
    if not cabi.is_built():
        pytest.skip("libwavernn_b200.so not built")
    return cabi.load()


@pytest.fixture(scope="module")
def win(lib):
    n = lib.wrnn_debug_resample_table(None)
    w = np.empty(n, dtype=np.float64)
    assert lib.wrnn_debug_resample_table(w.ctypes.data) == n
    return w


def host(lib, xs, rates, sr_out=SR):
    """wrnn_debug_resample on a batch: the list of outputs, each followed in memory by a sentinel that must survive."""
    xs = [np.ascontiguousarray(x, dtype=np.float32) for x in xs]
    bufs = [np.full(lib.wrnn_resample_length(x.size, r, sr_out) + 1, 7.0, dtype=np.float32) for x, r in zip(xs, rates)]
    arr, n = cabi.utt_array(cabi.WrnnResampleUtt,
                            [(x.ctypes.data, x.size, r, b.ctypes.data) for x, r, b in zip(xs, rates, bufs)])
    rc = lib.wrnn_debug_resample(arr, n, sr_out)
    assert rc == 0, lib.wrnn_last_error()
    assert all(b[-1] == 7.0 for b in bufs), "written past wrnn_resample_length"
    return [b[:-1] for b in bufs]


def signals(sr, n, seed=0):
    """Tones, a chirp, noise and a speech-like signal (a 120 Hz pulse train through two formant resonators, gated)."""
    import scipy.signal
    rs = np.random.RandomState(seed)
    t = np.arange(n) / sr
    nyq = min(sr, SR) / 2
    tones = 0.3 * np.sin(2 * np.pi * 440 * t) + 0.2 * np.sin(2 * np.pi * 0.41 * nyq * t + 1.0)
    chirp = 0.8 * scipy.signal.chirp(t, 50, t[-1] if n > 1 else 1.0, 0.95 * sr / 2)
    noise = 0.25 * rs.randn(n)
    pulses = (np.arange(n) % max(1, int(sr / 120)) == 0).astype(np.float64)
    speech = pulses
    for f, bw in ((700, 130), (1220, 70)):
        if f < sr / 2:
            r = np.exp(-np.pi * bw / sr)
            speech = scipy.signal.lfilter([1 - r], [1, -2 * r * np.cos(2 * np.pi * f / sr), r * r], speech)
    speech = 0.5 * speech / max(np.abs(speech).max(), 1e-9) * (np.sin(2 * np.pi * 3 * t) > -0.3)
    return {k: v.astype(np.float32) for k, v in (("tones", tones), ("chirp", chirp), ("noise", noise), ("speech", speech))}


def same_bits(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32))


def test_table_matches_design(win):
    """The library's half-window is resampy's sinc_window at p = 16 within 8 float64 ulps per entry (measured: median
    1, largest 7: glibc's sin and a long-double i0 series against numpy's sin and scipy's Cephes i0)."""
    ref = R.table()
    assert win.shape == ref.shape == (64 * 2 ** 16 + 1,)
    assert np.all(np.abs(win - ref) <= 8 * np.spacing(np.abs(ref)))


@pytest.mark.parametrize("sr", RATES)
def test_host_hook_matches_oracle(lib, win, sr):
    sig = signals(sr, sr // 4)
    got = host(lib, list(sig.values()), [sr] * len(sig))
    for (name, x), y in zip(sig.items(), got):
        assert same_bits(y, R.resample(x, sr, SR, win=win)), f"{name} at {sr} Hz"


@pytest.mark.parametrize("sr,n", [(8000, 1), (16000, 1), (44100, 2), (48000, 3), (16000, 40), (48000, 200), (44100, 127),
                                  (8000, 63), (22051, 5), (22050, 1)])
def test_edge_lengths(lib, win, sr, n):
    """n = 1, n shorter than the filter's half-width (64 zero crossings), and lengths whose last sample is librosa's zero
    padding."""
    x = np.random.RandomState(n).uniform(-1, 1, n).astype(np.float32)
    (y,) = host(lib, [x], [sr])
    ref = R.resample(x, sr, SR, win=win)
    assert same_bits(y, ref)
    n_out, n_len = R.output_length(n, sr, SR)
    assert y.size == (n if sr == SR else n_len)
    if sr != SR and n_len > n_out:
        assert y[-1] == 0.0


def test_padded_last_sample(lib, win):
    n = 1001                                            # 1001 * 22050 / 44100 = 500.5 -> 500 computed, 501 returned
    x = np.random.RandomState(3).uniform(-1, 1, n).astype(np.float32)
    (y,) = host(lib, [x], [44100])
    assert y.size == 501 and y[-1] == 0.0 and y[-2] != 0.0
    assert same_bits(y, R.resample(x, 44100, SR, win=win))


def test_batch_is_each_alone(lib):
    xs = [signals(sr, sr // 8, seed=i)["speech"] for i, sr in enumerate(RATES)]
    got = host(lib, xs, RATES)
    for x, sr, y in zip(xs, RATES, got):
        assert same_bits(y, host(lib, [x], [sr])[0])


def gain_bound(sr, peak):
    """The truncation of index_step = int(scale * 2^16) scales the filter's gain by scale * 2^16 / index_step."""
    scale = min(1.0, SR / sr)
    return peak * (scale * 2 ** 16 / int(scale * 2 ** 16) - 1)


@pytest.mark.parametrize("sr", (44100, 48000, 16000, 8000))
def test_oracle_against_analytic_tones(sr):
    t = np.arange(sr) / sr
    freqs = (440.0, 1234.5, 3000.0)
    x = sum(0.3 * np.sin(2 * np.pi * f * t) for f in freqs).astype(np.float32)
    y = R.resample(x, sr, SR)
    to = np.arange(y.size) / SR
    ref = sum(0.3 * np.sin(2 * np.pi * f * to) for f in freqs)
    core = slice(300, y.size - 300)
    assert np.abs(y[core] - ref[core]).max() <= 2e-6 + gain_bound(sr, 0.9)


@pytest.mark.parametrize("sr", (44100, 48000, 16000, 8000))
def test_oracle_against_torchaudio(sr):
    torch = pytest.importorskip("torch")
    TF = pytest.importorskip("torchaudio.functional")
    t = np.arange(sr) / sr
    x = (0.4 * np.sin(2 * np.pi * 523.25 * t) + 0.3 * np.sin(2 * np.pi * 2750.0 * t)).astype(np.float32)
    y = R.resample(x, sr, SR)
    ta = TF.resample(torch.from_numpy(x).double(), sr, SR, lowpass_filter_width=64, rolloff=R.ROLLOFF,
                     resampling_method="sinc_interp_kaiser", beta=R.BETA).numpy()
    L = min(y.size, ta.size)
    core = slice(300, L - 300)
    assert np.abs(y[core] - ta[core]).max() <= 2e-6 + gain_bound(sr, 0.7)


def test_stopband(lib):
    """A 15 kHz tone at 44.1 kHz lies above the new Nyquist frequency: less than 1e-5 of it survives (the p = 9
    restatement leaves 2.3e-7)."""
    sr = 44100
    x = (0.9 * np.sin(2 * np.pi * 15000 * np.arange(sr) / sr)).astype(np.float32)
    (y,) = host(lib, [x], [sr])
    assert np.abs(y[300:-300]).max() < 1e-5


def test_sequential_register():
    """resampy advances its time register by repeated addition; the library computes t * (1 / ratio) so that every
    output is independent.  On 10 s at 48 kHz the two differ by at most 4.3e-6 (rms 1.2e-7; DESIGN.md §3.10)."""
    sr = 48000
    rs = np.random.RandomState(1)
    t = np.arange(10 * sr) / sr
    x = (0.4 * np.sin(2 * np.pi * 220 * t) + 0.3 * np.sin(2 * np.pi * 3100 * t) + 0.05 * rs.randn(t.size)).astype(np.float32)
    a = R.resample(x, sr, SR)
    b = R.resample(x, sr, SR, sequential=True)
    d = np.abs(a.astype(np.float64) - b)
    assert d.max() <= 5e-6 and np.sqrt(np.mean(d ** 2)) <= 2e-7
    assert d.max() > 0                                  # the two registers do differ


def test_length(lib):
    for n, sr_in, sr_out in ((1, 8000, 22050), (1001, 44100, 22050), (441000, 44100, 22050), (48000, 48000, 22050),
                             (12345, 16000, 22050), (7, 22050, 22050), (0, 44100, 22050), (3, 22051, 22050)):
        want = n if sr_in == sr_out else R.output_length(n, sr_in, sr_out)[1]
        assert lib.wrnn_resample_length(n, sr_in, sr_out) == want
    assert lib.wrnn_resample_length(-1, 44100, 22050) == -1
    assert lib.wrnn_resample_length(10, 0, 22050) == -1
    assert lib.wrnn_resample_length(10, 44100, -5) == -1


def test_struct_layout():
    U = cabi.WrnnResampleUtt
    assert C.sizeof(U) == 32
    assert [getattr(U, f).offset for f in ("x", "n", "sample_rate", "pad", "y")] == [0, 8, 16, 20, 24]


def refusal(lib, utts, n=None, sr_out=SR):
    arr, k = cabi.utt_array(cabi.WrnnResampleUtt, utts)
    rc = lib.wrnn_debug_resample(arr, k if n is None else n, sr_out)
    return rc, (lib.wrnn_last_error() or b"").decode()


def test_refusals(lib):
    x = np.zeros(1000, np.float32)
    y = np.zeros(4000, np.float32)
    ok = (x.ctypes.data, 1000, 44100, y.ctypes.data)
    assert refusal(lib, [ok])[0] == cabi.WRNN_OK
    cases = [
        ([ok], 0, "n_utts >= 1"),
        ([], None, "n_utts >= 1"),
        ([ok, (0, 1000, 44100, y.ctypes.data)], None, "utterance 1: x and y are required"),
        ([ok, (x.ctypes.data, 1000, 44100, 0)], None, "utterance 1: x and y are required"),
        ([ok, ok, (x.ctypes.data, 1000, 0, y.ctypes.data)], None, "utterance 2: sample_rate must be > 0"),
        ([(x.ctypes.data, 1000, -8000, y.ctypes.data)], None, "utterance 0: sample_rate must be > 0"),
        ([ok, (x.ctypes.data, 0, 44100, y.ctypes.data)], None, "utterance 1: n must be >= 1"),
        ([(x.ctypes.data, 2, 48000, y.ctypes.data)], None, "utterance 0: n = 2 at 48000 Hz gives no output sample"),
        ([(x.ctypes.data, 2 ** 30, 2 ** 31 - 1, y.ctypes.data)], None, "utterance 0: the ratio 22050 / 2147483647 is below 2^-16"),
        ([(x.ctypes.data, 2 ** 30, 8000, y.ctypes.data)], None, "fewer than 2^31 output samples"),
        ([(x.ctypes.data, 2 ** 30, 22050, y.ctypes.data), (x.ctypes.data, 2 ** 30, 22050, y.ctypes.data)], None,
         "fewer than 2^31 output samples"),
    ]
    for utts, n, msg in cases:
        rc, err = refusal(lib, utts, n)
        assert rc == cabi.WRNN_E_INVALID and msg in err, (msg, err)
    rc, err = refusal(lib, [ok], sr_out=0)
    assert rc == cabi.WRNN_E_INVALID


def test_null_analysis_object(lib):
    x = np.zeros(10, np.float32)
    arr, n = cabi.utt_array(cabi.WrnnResampleUtt, [(x.ctypes.data, 10, 44100, x.ctypes.data)])
    assert lib.wrnn_resample_many(None, arr, n, None) == cabi.WRNN_E_INVALID
    assert lib.wrnn_resample_many_host(None, arr, n) == cabi.WRNN_E_INVALID
    assert "null analysis object" in lib.wrnn_last_error().decode()


def test_abi_version_unchanged(lib):
    assert lib.wrnn_abi_version() == 5 == cabi.ABI_VERSION
