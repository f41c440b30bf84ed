"""Griffin-Lim (wrnn_griffinlim_many) across every configuration wrnn_mel_create accepts, without a device
(tests/gl_edges.py's mels on tests/mel_edges.py's grid):

  1. The kernels' code run on the host (wrnn_debug_griffinlim) against the oracle (tests/gl_oracle.py) at n_iter 0, 1
     and 2 under the local measure gl_edges.local_steps; S within 1e-5 of its peak.
  2. Negative controls: each restatement in gl_edges.WRONG misses gl_edges.LOCAL_TOL somewhere on the grid, each in
     gl_edges.INVISIBLE stays inside it everywhere; an error the former peak-relative check cannot see is caught.
  3. The planner accepts the shortest T of every cell and refuses one frame less, naming the utterance.
  4. Out-of-range mels give the bits of the same mel clipped to [0, 1]; a NaN stays NaN where the oracle's does.
  5. On the oracle, spectral convergence falls from 0 to 8 iterations in every cell."""
import numpy as np
import pytest

import gl_edges as E
import gl_oracle as G
from test_gl_abi import ULPS_EARLY, gl_plan, host_gl
from wavernn_b200 import cabi


@pytest.fixture(scope="module")
def lib():
    if not cabi.is_built():
        import __graft_entry__ as g
        g.build()
    return cabi.load()


def bits(a):
    return np.ascontiguousarray(a).view(np.int32)


# ---- 1. the kernels' code on the host ---------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(E.GRID))
def test_kernel_code_on_the_host(lib, name):
    c = E.cfg(name)
    worst = {0: 0.0, 1: 0.0, 2: 0.0}
    for k, mel in E.mels(c).items():
        S_ref = G.mel_to_stft(mel, **c)
        for n_iter in (0, 1, 2):
            got, S = host_gl(lib, mel, E.SEED, n_iter, **c)
            if n_iter == 0:
                dS = np.abs(S - S_ref).max() / max(S_ref.max(), 1e-30)
                assert dS <= 1e-5, (k, dS)
            ref = E.oracle(mel, n_iter, **c)
            assert got.shape == ref.shape and np.isfinite(got).all(), (k, n_iter)
            d = float(E.local_steps(got, ref, c).max())
            worst[n_iter] = max(worst[n_iter], d)
            assert d <= E.LOCAL_TOL[n_iter], (k, n_iter, d)
    print(f"{name}: host run vs oracle, local float32 steps at n_iter 0/1/2: "
          + " / ".join(f"{worst[n]:.1f}" for n in (0, 1, 2)))


def test_restatement_defaults_equal_the_oracle():
    """The restatement the negative controls edit is the oracle, bit for bit, when nothing is edited."""
    for name in ("default", "fft4096-hop5000", "sr8k-fft256-mels128"):
        c = E.cfg(name)
        mel = E.mels(c)["shortest"]
        A, B = G.fb32(**c), G.amplitudes(mel, **c)
        assert np.array_equal(bits(E._solve(A, B)), bits(G.nnls_fista(A, B))), name
        for n_iter in (0, 2):
            assert np.array_equal(bits(E._restated(mel, n_iter, E.SEED, **c)), bits(E.oracle(mel, n_iter, **c))), name


# ---- 2. negative controls -----------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def restatement_gaps():
    """name -> (largest ratio of the local measure to LOCAL_TOL over the grid, its cell).  At hop_length 1 the speech
    and out-of-range mels only (a solve of 1,026 frames takes seconds)."""
    gaps = {k: (0.0, None) for k in list(E.WRONG) + list(E.INVISIBLE)}
    for name in E.GRID:
        c = E.cfg(name)
        ms = E.mels(c)
        if c["hop_length"] == 1:
            ms = {k: ms[k] for k in ("shortest", "out_of_range")}
        for k, mel in ms.items():
            refs = [E.oracle(mel, n_iter, **c) for n_iter in (0, 1, 2)]
            for w, f in {**E.WRONG, **E.INVISIBLE}.items():
                for n_iter, out in enumerate(f(mel, 2, E.SEED, stages=True, **c)):
                    r = float(E.local_steps(out, refs[n_iter], c).max()) / E.LOCAL_TOL[n_iter]
                    if r > gaps[w][0]:
                        gaps[w] = (r, f"{name}/{k}/n_iter={n_iter}")
    return gaps


@pytest.mark.parametrize("wrong", list(E.WRONG))
def test_wrong_restatement_misses_the_tolerance(restatement_gaps, wrong):
    r, cell = restatement_gaps[wrong]
    print(f"{wrong}: largest miss {r:.3g} x LOCAL_TOL at {cell}")
    assert r > 1


@pytest.mark.parametrize("invisible", list(E.INVISIBLE))
def test_invisible_slips_stay_inside_the_tolerance(restatement_gaps, invisible):
    """Documents what the output cannot show: these slips move no output by more than its own rounding."""
    r, cell = restatement_gaps[invisible]
    print(f"{invisible}: largest gap {r:.3g} x LOCAL_TOL at {cell}")
    assert r <= 1


def test_the_local_measure_sees_what_the_peak_measure_cannot():
    """Where the hop is longer than the window, the output's peak is a division by a window sum-square near 0, so 4
    float32 steps of the peak exceed the typical sample: tripling every sample at or below the median magnitude passes
    the former check (ULPS_EARLY steps of the peak) and fails the local one."""
    c = E.cfg("fft4096-hop5000")
    ref = E.oracle(E.mels(c)["speech"], 1, **c)
    a = np.abs(ref)
    med = np.median(a)
    bad = ref.copy()
    bad[a <= med] *= 3
    change = float(np.abs(bad - ref).max())
    old_tol = ULPS_EARLY * float(np.spacing(a.max()))
    local = float(E.local_steps(bad, ref, c).max())
    print(f"fft4096-hop5000: peak {a.max():.3g}, median |sample| {med:.3g}; change {change / med:.2f} medians, former "
          f"tolerance {old_tol / med:.2f} medians ({old_tol:.2g}); local measure {local:.3g} steps")
    assert E.peak_steps(bad, ref) <= ULPS_EARLY
    assert local > E.LOCAL_TOL[1]


# ---- 3. the planner ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(E.GRID))
def test_shortest_length_is_the_planners_limit(lib, name):
    c = E.cfg(name)
    T0 = E.shortest(c)
    assert c["hop_length"] * (T0 - 1) > c["n_fft"] // 2 >= c["hop_length"] * (T0 - 2)
    rc, msg, f0 = gl_plan(lib, [T0, T0 + 1], **c)
    assert rc == 0, msg
    assert list(f0[:3]) == [0, T0, 2 * T0 + 1]
    for Ts, at in (([T0 - 1], 0), ([T0, T0 - 1], 1)):
        rc, msg, _ = gl_plan(lib, Ts, **c)
        assert rc == cabi.WRNN_E_INVALID and f"utterance {at}: hop_length * (T - 1) must be > n_fft / 2" in msg, msg


# ---- 4. out-of-range and NaN mels --------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["default", "fft4096-hop5000", "sr16k-fmin7990", "db-20", "db-120", "mels1"])
def test_out_of_range_mel_is_clipped(lib, name):
    c = E.cfg(name)
    mel = E.mels(c)["out_of_range"]
    assert np.isinf(mel).any() and (mel == -1).any() and (mel == 2).any()
    for n_iter in (0, 2):
        got, S = host_gl(lib, mel, E.SEED, n_iter, **c)
        want, S_want = host_gl(lib, np.clip(mel, 0, 1), E.SEED, n_iter, **c)
        assert np.array_equal(bits(got), bits(want)) and np.array_equal(bits(S), bits(S_want)), n_iter
        assert np.isfinite(got).all()


@pytest.mark.parametrize("name", ["default", "win1", "fft512-hop600", "fft4096-hop5000", "sr16k-fmin7990"])
def test_nan_mel(lib, name):
    """A NaN value in a band with filter weight makes NaN exactly the samples the oracle's output has NaN (at n_iter 0,
    those the frame's n_fft samples cover: its window's zeros times NaN are NaN); every other sample stays within
    LOCAL_TOL.  (In a band without weight the kernels never read the value, where the oracle's 0 x NaN spreads it.)"""
    c = E.cfg(name)
    mel = E.mels(c)["speech"].copy()
    t = mel.shape[1] // 2
    mel[int(G.fb32(**c).sum(axis=1).argmax()), t] = np.nan
    N, hop = c["n_fft"], c["hop_length"]
    for n_iter in (0, 1):
        got, _ = host_gl(lib, mel, E.SEED, n_iter, **c)
        with np.errstate(invalid="ignore"):
            ref = E.oracle(mel, n_iter, **c)
        assert np.isnan(got).any() and np.array_equal(np.isnan(got), np.isnan(ref)), n_iter
        if n_iter == 0:
            p = np.arange(got.size) + N // 2
            assert np.array_equal(np.isnan(got), (p >= t * hop) & (p < t * hop + N))
        assert E.local_steps(got, ref, c).max() <= E.LOCAL_TOL[n_iter], n_iter


# ---- 5. convergence -----------------------------------------------------------------------------------------------------
# ||stft(y)| - S| / |S| on the oracle after 8 iterations, over the same after none, on each cell's speech mel (the
# shortest at hop_length 1): measured 0.115 (win3) to 0.485 (fft512-hop600), except sr16k-fmin7990, whose 80 bands
# share the 10 Hz below the Nyquist frequency (0.853 -> 0.848: with S nearly empty, little is there to converge to).
SC_RATIO = 0.5
SC_RATIO_NEAR_NYQUIST = 1.0                    # sr16k-fmin7990: it must still fall


@pytest.mark.parametrize("name", list(E.GRID))
def test_spectral_convergence_falls(name):
    c = E.cfg(name)
    m = E.mels(c)
    mel = m.get("speech", m["shortest"])
    S = E.magnitudes(mel, **c)
    sc = [G.spectral_convergence(E.oracle(mel, n, **c), S, **c) for n in (0, 8)]
    print(f"{name}: spectral convergence {sc[0]:.3f} -> {sc[1]:.3f} ({sc[1] / sc[0]:.3f})")
    assert sc[1] < (SC_RATIO_NEAR_NYQUIST if name == "sr16k-fmin7990" else SC_RATIO) * sc[0]
