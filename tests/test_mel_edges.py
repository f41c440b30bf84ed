"""The mel analysis across every configuration wrnn_mel_create accepts, without a device (tests/mel_edges.py's grid):

  1. The oracle (tests/mel_oracle.py) against torch's STFT and torchaudio's filterbank at the pinned grid points
     (tests/golden/mel_pins.npz): the STFT and dB path to one output step, the filterbank at torchaudio's float32.
  2. The tables wrnn_mel_create builds: the window bit for bit, the filterbank to float64 precision, the band ranges.
  3. The kernel's per-frame code run on the host (wrnn_debug_mel_frames) against the oracle at MEL_TOL on every grid
     point and signal, digital silence at its exact value, and against the pins.
  4. Negative controls: each wrong restatement in mel_edges.WRONG misses MEL_TOL somewhere on the grid.
  5. Non-finite samples: NaN makes exactly the frames that read it NaN, as the restatement does (empty bands
     excepted), and ±inf never leaves a band with filter weight finite below 1."""
import ctypes

import numpy as np
import pytest

import helpers
import mel_edges as ME
import mel_oracle as MO
from test_mel_abi import MEL_TOL
from wavernn_b200 import cabi

# Per pinned array: (filterbank, max |weight difference| over the largest weight; mel through the oracle's own
# filterbank, absolute).  torchaudio builds its filterbank in float32, which sets both: the bounds are about 2 x the
# gaps measured (in the comments).  Through the pin's own filterbank the oracle lands within MEL_TOL everywhere.
PIN_BOUNDS = {
    "default": (1e-5, 4e-6),            # 4.3e-6, 1.07e-6
    "win1": (1e-5, MEL_TOL),             # 4.3e-6, 6.0e-8
    "win1101": (1e-5, 2.5e-6),           # 4.3e-6, 1.01e-6
    "fft256-mels128": (1.2e-5, 4.5e-5),  # 5.9e-6, 2.1e-5: narrow bands near the floor
    "sr16k-fmin2000": (2.7e-5, 4.5e-6),  # 1.3e-5, 2.0e-6
    "sr44k": (3.5e-6, 3.5e-6),           # 1.6e-6, 1.5e-6
    "db-120": (1e-5, 2e-6),              # 4.3e-6, 8.3e-7
}


@pytest.fixture(scope="module")
def lib():
    if not cabi.is_built():
        import __graft_entry__ as g
        g.build()
    return cabi.load()


def pin_input(p, name):
    """The waveform the pin at grid point `name` analysed, and its key suffix in mel_pins.npz."""
    if name == "default":
        return helpers.load_golden("trained_tacotron.npz")["wav"].astype(np.float32), ""
    key = f"y_{name}"
    y = p[key] if key in p.files else helpers.load_golden("trained_tacotron.npz")["wav"].astype(np.float32)
    return y, "_" + name


def host_frames(lib, y, c):
    y = np.ascontiguousarray(y, dtype=np.float32)
    out = np.full((c["n_mels"], 1 + y.size // c["hop_length"]), -7.0, dtype=np.float32)
    rc = lib.wrnn_debug_mel_frames(ctypes.byref(cabi.mel_cfg(**c)), y.ctypes.data, y.size, out.ctypes.data)
    assert rc == 0, lib.wrnn_last_error().decode()
    return out


def host_tables(lib, c):
    nb = c["n_fft"] // 2 + 1
    win, basis = np.zeros(c["n_fft"]), np.zeros((c["n_mels"], nb))
    bands = np.zeros((c["n_mels"], 2), dtype=np.int32)
    assert lib.wrnn_debug_mel_tables(ctypes.byref(cabi.mel_cfg(**c)), win.ctypes.data, basis.ctypes.data,
                                     bands.ctypes.data) == 0
    return win, basis, bands


def reads(y, c, pred):
    """[T] bool: the frames whose n_fft padded samples include one where pred(sample) holds (reflected copies too)."""
    half, hop = c["n_fft"] // 2, c["hop_length"]
    yp = np.pad(pred(np.asarray(y)), half, mode="reflect")
    T = 1 + y.size // hop
    return yp[np.arange(c["n_fft"])[:, None] + hop * np.arange(T)[None]].any(axis=0)


# ---- 1. the oracle against the independent pins --------------------------------------------------------------------
@pytest.mark.parametrize("name", list(PIN_BOUNDS))
def test_oracle_matches_pins(name):
    p = helpers.load_golden("mel_pins.npz")
    c = ME.cfg(name)
    y, key = pin_input(p, name)
    fb_bound, mel_bound = PIN_BOUNDS[name]
    fb = p["fbank" + key].astype(np.float64)
    d_fb = np.abs(MO.mel_basis(**c) - fb).max() / fb.max()
    d_mel = np.abs(MO.melspectrogram(y, **c) - p["mel" + key]).max()
    M = fb @ MO.magnitudes(y, **c).astype(np.float64)           # the oracle's STFT through the pin's own filterbank
    own = np.clip((20 * np.log10(np.maximum(1e-5, M)) - c["min_level_db"]) / -c["min_level_db"], 0, 1).astype(np.float32)
    d_own = np.abs(own - p["mel" + key]).max()
    print(f"{name}: oracle vs torch/torchaudio: filterbank {d_fb:.2e} of the largest weight (bound {fb_bound:.1e}), "
          f"mel {d_mel:.2e} (bound {mel_bound:.1e}), mel through the pin's filterbank {d_own:.2e}")
    assert p["mel" + key].shape == (c["n_mels"], 1 + y.size // c["hop_length"])
    assert d_fb <= fb_bound and d_mel <= mel_bound and d_own <= MEL_TOL


def test_one_sample_window_pin():
    """torch.hann_window(1, periodic=True) is [1], as scipy's get_window('hann', 1) is: the window is not the
    formula's 0.5 + 0.5 cos(-pi) = 0."""
    w = helpers.load_golden("mel_pins.npz")["window_win1"]
    assert np.array_equal(w, MO.window(2048, 1)) and w.sum() == 1.0 and w[1023] == 1.0


# ---- 2. the host tables ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(ME.GRID))
def test_host_tables(lib, name):
    """Window bit for bit; each band's weights within 1e-12 of its peak weight, or of the float64 conditioning of a
    narrow triangle where that is larger (a weight is (f_k - f_lo) / (f_mid - f_lo) x enorm: one rounding of the band
    edges, about 2^-52 f_hi, moves it by 2^-52 f_hi / min(f_mid - f_lo, f_hi - f_mid) x enorm); the same nonzero
    ranges."""
    c = ME.cfg(name)
    win, basis, bands = host_tables(lib, c)
    assert np.array_equal(win, MO.window(**c))
    ref = MO.mel_basis(**c)
    mel_f = MO.mel_to_hz(np.linspace(MO.hz_to_mel(c["fmin"]), MO.hz_to_mel(c["sample_rate"] / 2), c["n_mels"] + 2))
    worst = 0.0
    for m in range(c["n_mels"]):
        lo, mid, hi = mel_f[m:m + 3]
        cond = 2.0 ** -52 * hi / min(mid - lo, hi - mid) * 2.0 / (hi - lo)
        tol = max(1e-12 * ref[m].max(), 4 * cond)
        d = np.abs(basis[m] - ref[m]).max()
        worst = max(worst, d / tol)
        assert d <= tol, (m, d, tol)
        nz = np.flatnonzero(basis[m] > 0)
        assert np.array_equal(nz, np.flatnonzero(ref[m] > 0)), m
        lo_k, cnt = bands[m]
        assert cnt == nz.size and (cnt == 0 or (lo_k == nz[0] and nz[-1] == lo_k + cnt - 1)), m
    empty = int((ref.max(axis=1) == 0).sum())
    print(f"{name}: filterbank worst {worst:.2f} of its bound, {empty} empty bands")


# ---- 3. the kernel's code on the host ----------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(ME.GRID))
def test_kernel_code_on_the_host(lib, name):
    c = ME.cfg(name)
    worst = {}
    for k, y in ME.signals(c).items():
        got, ref = host_frames(lib, y, c), MO.melspectrogram(y, **c)
        assert got.shape == ref.shape, k
        worst[k] = float(np.abs(got - ref).max())
        if k == "silence_click":
            silent = ~reads(y, c, lambda v: v != 0)
            assert silent.sum() >= 1
            assert (got[:, silent] == ME.silent_value(c["min_level_db"])).all()
            assert (ref[:, silent] == ME.silent_value(c["min_level_db"])).all()
    print(f"{name}: host run of the kernel code vs oracle, worst {max(worst.values()):.3e} "
          + " ".join(f"{k} {v:.1e}" for k, v in worst.items()))
    assert max(worst.values()) <= MEL_TOL, worst


@pytest.mark.parametrize("L", [-20.0, -37.5, -100.0, -120.0])
def test_silence_value(lib, L):
    """Digital silence is float32(clip((-100 - L) / -L, 0, 1)) exactly in every band: 0 at -100 dB and above, 1/6
    at -120."""
    c = dict(MO.DEFAULT, min_level_db=L)
    want = ME.silent_value(L)
    got = host_frames(lib, np.zeros(5000, np.float32), c)
    assert (got == want).all() and (MO.melspectrogram(np.zeros(5000, np.float32), **c) == want).all()
    assert want == (np.float32(1 / 6) if L == -120.0 else np.float32(0))


@pytest.mark.parametrize("name", [n for n in PIN_BOUNDS if n != "default"])
def test_kernel_code_matches_pins(lib, name):
    p = helpers.load_golden("mel_pins.npz")
    y, key = pin_input(p, name)
    d = np.abs(host_frames(lib, y, ME.cfg(name)) - p["mel" + key]).max()
    print(f"{name}: host run of the kernel code vs torch/torchaudio {d:.2e}")
    assert d <= PIN_BOUNDS[name][1]


# ---- 4. negative controls ---------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def restatement_gaps():
    """name -> (largest gap from the oracle over the grid and the grid's signals, its cell)."""
    gaps = {k: (0.0, None) for k in list(ME.WRONG) + list(ME.INVISIBLE)}
    for name in ME.GRID:
        c = ME.cfg(name)
        for s, y in ME.signals(c).items():
            ref = MO.melspectrogram(y, **c)
            for k, f in {**ME.WRONG, **ME.INVISIBLE}.items():
                d = float(np.abs(f(y, **c) - ref).max())
                if d > gaps[k][0]:
                    gaps[k] = (d, f"{name}/{s}")
    return gaps


@pytest.mark.parametrize("wrong", list(ME.WRONG))
def test_wrong_restatement_misses_the_tolerance(restatement_gaps, wrong):
    d, cell = restatement_gaps[wrong]
    print(f"{wrong}: largest miss {d:.3e} = {d / MEL_TOL:.3g} x MEL_TOL at {cell}")
    assert d > MEL_TOL


@pytest.mark.parametrize("invisible", list(ME.INVISIBLE))
def test_invisible_slips_stay_inside_the_tolerance(restatement_gaps, invisible):
    """Documents what the output cannot show: these slips move no output by more than its own rounding."""
    d, cell = restatement_gaps[invisible]
    print(f"{invisible}: largest gap {d:.3e} at {cell}")
    assert d <= MEL_TOL


# ---- 5. non-finite samples --------------------------------------------------------------------------------------------
NONFINITE_GRID = ["default", "win1", "win2048", "fft256-mels128", "fft512-hop600", "sr16k-fmin7990", "db-120"]


def bad_positions(n):
    return {"first": [0], "second": [1], "mid": [n // 2], "last": [n - 1], "two": [3, n - 2]}


@pytest.mark.parametrize("name", NONFINITE_GRID)
def test_nan_samples(lib, name):
    """A NaN sample makes every frame that reads it (reflected copies included) NaN in every band with filter weight,
    as the restatement does; a band without weight keeps its silent value (numpy's 0 x NaN makes it NaN); every other
    frame equals the oracle."""
    c = ME.cfg(name)
    y0 = ME.signals(c)["noise"]
    has_weight = MO.mel_basis(**c).max(axis=1) > 0
    for where, idx in bad_positions(y0.size).items():
        y = y0.copy()
        y[idx] = np.nan
        got, ref = host_frames(lib, y, c), MO.melspectrogram(y, **c)
        bad = reads(y, c, np.isnan)
        assert np.array_equal(np.isnan(ref).any(axis=0), bad) and np.isnan(ref[:, bad]).all(), where
        if c["hop_length"] <= c["n_fft"] // 2:
            assert bad.any(), where
        assert np.array_equal(np.isnan(got), np.outer(has_weight, bad)), where
        assert (got[~has_weight][:, bad] == ME.silent_value(c["min_level_db"])).all(), where
        assert np.abs(got[:, ~bad] - ref[:, ~bad]).max(initial=0) <= MEL_TOL, where


@pytest.mark.parametrize("name", NONFINITE_GRID)
def test_inf_samples(lib, name):
    """±inf: which bins turn inf and which NaN depends on the FFT's order, so only this is required: no band with
    filter weight in a frame that reads the sample is finite below 1, and every other frame equals the oracle."""
    c = ME.cfg(name)
    y0 = ME.signals(c)["noise"]
    has_weight = MO.mel_basis(**c).max(axis=1) > 0
    for sign in (1, -1):
        for where, idx in bad_positions(y0.size).items():
            y = y0.copy()
            y[idx] = sign * np.inf
            with np.errstate(invalid="ignore"):   # inf - inf and 0 x inf inside the restatement's FFT and sums
                got, ref = host_frames(lib, y, c), MO.melspectrogram(y, **c)
            bad = reads(y, c, np.isinf)
            sub = got[has_weight][:, bad]
            assert not (np.isfinite(sub) & (sub < 1)).any(), (sign, where)
            assert np.abs(got[:, ~bad] - ref[:, ~bad]).max(initial=0) <= MEL_TOL, (sign, where)
