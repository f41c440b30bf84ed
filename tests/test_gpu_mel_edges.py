"""The mel analysis and the front end of wrnn_score_wav_many at their edges, on the GPU.

  1. The kernel on every grid point and signal of tests/mel_edges.py, in one guarded batch per configuration: against
     the oracle at test_mel_abi.MEL_TOL, against the torch/torchaudio pins, digital silence at its exact value.  Each
     recording sits between at least n_fft NaN samples and each mel between sentinel words, so a read outside [0, n)
     turns a frame NaN and a stray write breaks a sentinel: the guarded batch equals an unguarded one bit for bit.  How
     many values differ from the host run of the same code is reported, not asserted (device FMAs may move a rounding).
  2. About 2,000 utterances of mixed lengths (T = 1 included) in one launch, in two orders: each bit-identical to the
     utterance analysed alone; the host entry bit-identical to the device entry.
  3. Two batches on two streams sharing one analysis object equal the same batches run one after the other.
  4. wrnn_score_wav_many's front end: the peak at chosen indices and residues modulo 256 (the peak kernel's stride),
     negative, exactly 1.0 and one ulp above; the normalised recording and the MoL / linear targets equal the
     restatement bit for bit, and the losses equal wrnn_score_many of that mel and those targets (persistent fp16 MoL,
     persistent RAW mu-law).  The device quantiser equals the host's on every float32 in [-1, 1] (MoL 16-bit, RAW 9-bit
     linear) and, for mu-law (9 and 10 bits), on every float32 within 16 ulps of each code boundary plus 2^24 random
     inputs.
  5. Isolation: a recording with a NaN sample and an all-zero recording under peak_norm (0 / 0), batched between two
     clean recordings, leave the clean losses bit-identical.  Pinned: the NaN sample's own loss is NaN and no other
     loss of its recording is; every loss of the all-zero recording is NaN.
Run on a GPU: pytest -m gpu -s tests/test_gpu_mel_edges.py"""
import concurrent.futures
import os

import numpy as np
import pytest
import torch

import helpers
import mel_edges as ME
import mel_oracle as MO
from test_gpu_mel import composed, score_wav_device
from test_mel_abi import MEL_TOL
from test_mel_edges import PIN_BOUNDS, host_frames, pin_input
from wavernn_b200 import cabi

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
SENTINEL = 0x7FA5A5A5            # a NaN payload no arithmetic produces
GUARD = 64                       # sentinel words on each side of each mel


def bits(a):
    return np.ascontiguousarray(a).view(np.int32)


def analyse(an, ys, guard=False):
    """One wrnn_melspectrogram_many batch over device copies of ys; returns the host mels (and, guarded, whether every
    sentinel survived).  Guarded: the recordings sit in one buffer, each between n_fft NaN samples (n_fft + 64 after
    the last), and the mels in another, each between GUARD sentinel words."""
    if not guard:
        dms, _ = enqueue(an, ys, torch.cuda.current_stream(DEV))
        torch.cuda.synchronize(DEV)
        return [m.cpu().numpy() for m in dms]
    c = an.cfg
    Ts = [an.frames(y.size) for y in ys]
    pad = c.n_fft
    offs = np.cumsum([0] + [y.size + pad for y in ys])
    dy = torch.full((int(offs[-1]) + pad + 64,), float("nan"), device=DEV)
    for o, y in zip(offs, ys):
        dy[o + pad:o + pad + y.size].copy_(torch.as_tensor(y))
    moffs = np.cumsum([0] + [c.n_mels * T + GUARD for T in Ts])
    dm = torch.full((int(moffs[-1]) + GUARD,), SENTINEL, dtype=torch.int32, device=DEV)
    an.melspectrogram_many(ys=[dy.data_ptr() + 4 * int(o + pad) for o in offs[:-1]], ns=[y.size for y in ys],
                           mels=[dm.data_ptr() + 4 * int(o + GUARD) for o in moffs[:-1]],
                           stream=torch.cuda.current_stream(DEV).cuda_stream)
    torch.cuda.synchronize(DEV)
    h = dm.cpu().numpy()
    mels = [h[o + GUARD:o + GUARD + c.n_mels * T].view(np.float32).reshape(c.n_mels, T) for o, T in zip(moffs, Ts)]
    keep = np.ones(h.size, bool)
    for o, T in zip(moffs, Ts):
        keep[o + GUARD:o + GUARD + c.n_mels * T] = False
    return mels, bool((h[keep] == SENTINEL).all())


def enqueue(an, ys, st):
    """wrnn_melspectrogram_many on stream st over device copies of ys, without waiting: (device mels, device inputs)."""
    with torch.cuda.stream(st):
        dys = [torch.as_tensor(y).to(DEV) for y in ys]
        dms = [torch.full((an.cfg.n_mels, an.frames(y.size)), float("nan"), device=DEV) for y in ys]
        an.melspectrogram_many(ys=[y.data_ptr() for y in dys], ns=[y.size for y in ys], mels=[m.data_ptr() for m in dms],
                               stream=st.cuda_stream)
    return dms, dys


# ---- 1. the grid -----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def grid_worst():
    return {}


@pytest.mark.parametrize("name", list(ME.GRID))
def test_kernel_on_the_grid(lib, grid_worst, name):
    c = ME.cfg(name)
    an = cabi.MelAnalysis(**c)
    try:
        sigs = ME.signals(c)
        ys = list(sigs.values())
        p = helpers.load_golden("mel_pins.npz")
        if name in PIN_BOUNDS:
            ys.append(pin_input(p, name)[0])
        guarded, intact = analyse(an, ys, guard=True)
        plain = analyse(an, ys)
        assert intact, "a write outside a mel"
        worst, moved = {}, 0
        for k, y, g, u in zip(list(sigs) + ["pin"], ys, guarded, plain):
            assert np.array_equal(bits(g), bits(u)), (k, "guarded != unguarded")
            assert not np.isnan(g).any(), (k, "a read outside [0, n)")
            if k == "pin":
                d = float(np.abs(g - p["mel" + pin_input(p, name)[1]]).max())
                print(f"{name}: kernel vs torch/torchaudio pin {d:.2e} (bound {PIN_BOUNDS[name][1]:.1e})")
                assert d <= PIN_BOUNDS[name][1]
                continue
            ref = MO.melspectrogram(y, **c)
            worst[k] = float(np.abs(g - ref).max())
            moved += int((g != host_frames(lib, y, c)).sum())
            if k == "silence_click":
                silent = ~np.pad(y != 0, c["n_fft"] // 2, mode="reflect")[
                    np.arange(c["n_fft"])[:, None] + c["hop_length"] * np.arange(g.shape[1])[None]].any(axis=0)
                assert (g[:, silent] == ME.silent_value(c["min_level_db"])).all()
        grid_worst[name] = max(worst.values())
        print(f"{name}: max |kernel - oracle| {grid_worst[name]:.3e} over {len(worst)} signals; {moved} values differ "
              f"from the host run; guards and sentinels intact")
        assert grid_worst[name] <= MEL_TOL, worst
    finally:
        an.close()


def test_grid_maximum(grid_worst):
    if len(grid_worst) < len(ME.GRID):
        pytest.skip("the grid did not run whole")
    name = max(grid_worst, key=grid_worst.get)
    print(f"kernel vs oracle over the grid: {grid_worst[name]:.3e} = {grid_worst[name] / 2 ** -24:.2f} x 2^-24 "
          f"(at {name}); MEL_TOL = 2^-23")
    assert grid_worst[name] <= MEL_TOL


# ---- 2. large batches ---------------------------------------------------------------------------------------------------
def test_two_thousand_utterances_in_one_launch():
    c = ME.cfg("fft512-hop600")              # hop > n_fft / 2 + 1, so that T = 1 is reachable
    an = cabi.MelAnalysis(**c)
    try:
        rs = np.random.RandomState(5)
        grid_ns = [y.size for y in ME.signals(c).values()]   # 257 (min), 599 (T = 1), multiples of hop and one short
        ns = [grid_ns[i % len(grid_ns)] if i % 3 else int(rs.randint(257, 9000)) for i in range(2000)]
        ys = [(0.3 * rs.randn(n)).astype(np.float32) for n in ns]
        assert min(an.frames(n) for n in ns) == 1
        batch = analyse(an, ys)
        perm = rs.permutation(len(ys))
        pb = analyse(an, [ys[i] for i in perm])
        for k, i in enumerate(perm):
            assert np.array_equal(bits(pb[k]), bits(batch[i])), i
        for i, y in enumerate(ys):
            assert np.array_equal(bits(analyse(an, [y])[0]), bits(batch[i])), i
        host = an.melspectrogram_many_host(ys)
        assert all(np.array_equal(bits(a), bits(b)) for a, b in zip(host, batch))
        print(f"2000 utterances, {sum(an.frames(n) for n in ns)} frames: both orders, each alone and the host entry "
              "bit-identical")
    finally:
        an.close()


def test_two_streams_share_one_analysis():
    an = cabi.MelAnalysis()
    try:
        rs = np.random.RandomState(9)
        a = [(0.3 * rs.randn(int(n))).astype(np.float32) for n in rs.randint(1025, 60000, 40)]
        b = [np.clip(rs.randn(int(n)), -1, 1).astype(np.float32) for n in rs.randint(1025, 60000, 40)]
        want_a, want_b = analyse(an, a), analyse(an, b)
        s1, s2 = torch.cuda.Stream(DEV), torch.cuda.Stream(DEV)
        torch.cuda.synchronize(DEV)
        for _ in range(3):
            da, ia = enqueue(an, a, s1)
            db, ib = enqueue(an, b, s2)
            torch.cuda.synchronize(DEV)
            assert all(np.array_equal(bits(m.cpu().numpy()), bits(w)) for m, w in zip(da, want_a))
            assert all(np.array_equal(bits(m.cpu().numpy()), bits(w)) for m, w in zip(db, want_b))
    finally:
        an.close()


# ---- 4. the front end of wrnn_score_wav_many ----------------------------------------------------------------------------
def front_end(y, mode, n_classes, peak_norm, mu_law):
    """wrnn_debug_score_wav_targets on a device copy of y: (yn, x, peak) on the host."""
    lib, s = cabi.load(), torch.cuda.current_stream(DEV).cuda_stream
    dy = torch.as_tensor(y).to(DEV)
    yn, x, peak = torch.empty_like(dy), torch.empty_like(dy), torch.empty(1, device=DEV)
    assert lib.wrnn_debug_score_wav_targets(dy.data_ptr(), y.size, mode, n_classes, int(peak_norm), int(mu_law),
                                            yn.data_ptr(), x.data_ptr(), peak.data_ptr(), s) == 0
    torch.cuda.synchronize(DEV)
    return yn.cpu().numpy(), x.cpu().numpy(), float(peak.cpu()[0])


def peak_cases(n=6000):
    """name -> (recording, peak_norm): the peak at chosen indices and residues modulo 256, negative, exactly 1.0
    without peak_norm (left as it is) and one ulp above 1 (normalised)."""
    rs = np.random.RandomState(21)
    base = (0.4 * np.tanh(rs.randn(n))).astype(np.float32)
    cases = {}
    for i in (0, n - 1, 255, 256, 257, 511, 1000, 4097):
        y = base.copy()
        y[i] = np.float32(0.75)
        cases[f"peak@{i}"] = (y, True)
    y = base.copy()
    y[3001] = np.float32(-0.9)
    cases["negative@3001"] = (y, True)
    y = base.copy()
    y[777] = np.float32(1.0)
    cases["exactly1-no-norm"] = (y, False)
    y = base.copy()
    y[778] = np.nextafter(np.float32(1), np.float32(2))
    cases["above1-no-norm"] = (y, False)
    return cases


@pytest.mark.parametrize("head,mu_law", [("MOL", False), ("RAW", True)], ids=["MOL-fp16", "RAW-mu"])
def test_score_wav_front_end(head, mu_law):
    m = helpers.make_model(0, head)
    eng = cabi.Engine(m.hot_state(), n_classes=m.n_classes, mode=head, precision="fp16", engine="tcgen05")
    an = cabi.MelAnalysis()
    lib = cabi.load()
    try:
        eng.attach_upsampler(m.state_dict())
        mode, nc = (0, 30) if head == "MOL" else (1, m.n_classes)
        b = 16 if head == "MOL" else int(np.log2(m.n_classes))
        for name, (y, peak_norm) in peak_cases().items():
            want_yn = MO.normalise(y, peak_norm)
            assert np.abs(want_yn).max() == 1.0 or (name == "exactly1-no-norm" and np.array_equal(want_yn, y))
            yn, x, peak = front_end(y, mode, nc, peak_norm, mu_law)
            assert peak == np.abs(y).max(), name
            assert np.array_equal(bits(yn), bits(want_yn)), name
            host_x = np.empty_like(yn)
            lib.wrnn_debug_wav_targets(want_yn.ctypes.data, want_yn.size, mode, nc, int(mu_law), host_x.ctypes.data)
            assert np.array_equal(bits(x), bits(host_x)), name
            for lin_mode, lin_nc, lin_b in ((0, 30, 16), (1, 512, 9)):   # the MoL and linear labels: the restatement
                _, xl, _ = front_end(y, lin_mode, lin_nc, peak_norm, False)
                assert np.array_equal(bits(xl), bits(MO.targets(want_yn, "MOL" if lin_mode == 0 else "RAW", lin_b))), name
        ys = [c[0] for c in peak_cases().values()]
        for peak_norm in (False, True):
            got = score_wav_device(eng, an, ys, peak_norm, mu_law)
            ref, _ = composed(eng, an, ys, peak_norm, mu_law)
            assert all(np.array_equal(bits(a), bits(r)) for a, r in zip(got, ref)), peak_norm
        print(f"{head}: {len(ys)} peak cases: yn and targets bit-identical to the restatement, losses to score_many")
    finally:
        an.close()
        eng.close()


def ordered(f):
    """float32 -> an int64 that orders as the floats do (-0.0 and +0.0 both 0)."""
    i = np.asarray(f, np.float32).view(np.int32).astype(np.int64)
    return np.where(i < 0, -(i & 0x7FFFFFFF), i)


def unordered(k):
    k = np.asarray(k, np.int64)
    return np.where(k < 0, (-k) | 0x80000000, k).astype(np.uint32).view(np.float32)


def host_targets(lib, y, mode, nc, mu_law, workers=None):
    """wrnn_debug_wav_targets over y, split across threads (ctypes releases the GIL)."""
    x = np.empty_like(y)
    parts = np.array_split(np.arange(y.size), workers or os.cpu_count() or 1)
    def run(ix):
        if ix.size:
            lib.wrnn_debug_wav_targets(y[ix[0]:].ctypes.data, ix.size, mode, nc, int(mu_law), x[ix[0]:].ctypes.data)
    with concurrent.futures.ThreadPoolExecutor(len(parts)) as ex:
        list(ex.map(run, parts))
    return x


def device_targets(y_dev, mode, nc, mu_law):
    lib, s = cabi.load(), torch.cuda.current_stream(DEV).cuda_stream
    yn, x, peak = torch.empty_like(y_dev), torch.empty_like(y_dev), torch.empty(1, device=DEV)
    assert lib.wrnn_debug_score_wav_targets(y_dev.data_ptr(), y_dev.numel(), mode, nc, 0, int(mu_law), yn.data_ptr(),
                                            x.data_ptr(), peak.data_ptr(), s) == 0
    return x


QUANT = [("MOL", 16, False), ("RAW", 9, False), ("RAW", 9, True), ("RAW", 10, True)]


@pytest.mark.parametrize("head,b,mu_law", QUANT, ids=[f"{h}-{b}-{'mu' if u else 'lin'}" for h, b, u in QUANT])
def test_device_quantiser_equals_host(head, b, mu_law):
    lib = cabi.load()
    mode, nc = (0, 30) if head == "MOL" else (1, 2 ** b)
    lo, hi = int(ordered(np.float32(-1))), int(ordered(np.float32(1)))
    mismatches, covered = 0, 0
    if not mu_law:   # every float32 in [-1, 1]: each chunk of the bit patterns of [0, 1] and its negation
        chunk, one = 1 << 27, int(np.float32(1).view(np.int32))
        for k0 in range(0, one + 1, chunk):
            k1 = min(one + 1, k0 + chunk)
            pos = torch.arange(k0, k1, dtype=torch.int32, device=DEV).view(torch.float32)
            y_dev = torch.cat([pos, -pos])
            x_dev = device_targets(y_dev, mode, nc, False).cpu().numpy()
            y = y_dev.cpu().numpy()
            mismatches += int((bits(x_dev) != bits(host_targets(lib, y, mode, nc, False))).sum())
            covered += y.size
        what = "every float32 in [-1, 1]"
    else:            # every float32 within 16 ulps of each code boundary, found by bisection, plus 2^24 random inputs
        codes = 2 ** b
        levels = (np.float32(2) * np.arange(1, codes, dtype=np.float32)) / np.float32(codes - 1) - np.float32(1)
        a, z = np.full(codes - 1, lo), np.full(codes - 1, hi)   # the first float32 whose target reaches each level
        while (z - a > 1).any():
            mid = (a + z) // 2
            t = host_targets(lib, unordered(mid), mode, nc, True, workers=1)
            a, z = np.where(t >= levels, a, mid), np.where(t >= levels, mid, z)
        near = (z[:, None] + np.arange(-16, 17)[None]).reshape(-1)
        rs = np.random.RandomState(b)
        y = np.concatenate([unordered(np.clip(near, lo, hi)), unordered(rs.randint(lo, hi + 1, 1 << 24))])
        x_dev = device_targets(torch.from_numpy(y).to(DEV), mode, nc, True).cpu().numpy()
        mismatches = int((bits(x_dev) != bits(host_targets(lib, y, mode, nc, True))).sum())
        covered = y.size
        what = f"every float32 within 16 ulps of the {codes - 1} code boundaries plus 2^24 random inputs"
    print(f"{head}-{b}-{'mu' if mu_law else 'lin'} quantiser: {covered} inputs ({what}), {mismatches} mismatches")
    assert mismatches == 0


# ---- 5. isolation ---------------------------------------------------------------------------------------------------------
def test_bad_recordings_are_isolated():
    m = helpers.make_model(0, "MOL")
    eng = cabi.Engine(m.hot_state(), n_classes=30, mode="MOL", precision="fp16", engine="tcgen05")
    an = cabi.MelAnalysis()
    try:
        eng.attach_upsampler(m.state_dict())
        s = helpers.load_golden("trained_tacotron.npz")["wav"].astype(np.float32)
        clean = [s[:9000].copy(), s[20000:26500].copy()]
        nan_rec = s[10000:17000].copy()
        bad_at = 3333
        nan_rec[bad_at] = np.nan
        zero = np.zeros(6000, np.float32)
        ref = score_wav_device(eng, an, clean, True, False)
        got = score_wav_device(eng, an, [clean[0], nan_rec, zero, clean[1]], True, False)
        assert np.array_equal(bits(got[0]), bits(ref[0])) and np.array_equal(bits(got[3]), bits(ref[1]))
        nan_loss, zero_loss = np.isnan(got[1]), np.isnan(got[2])
        print(f"NaN sample at {bad_at} of {nan_rec.size}: losses NaN at {np.flatnonzero(nan_loss)[:8]} "
              f"({int(nan_loss.sum())} samples); all-zero recording under peak_norm: {int(zero_loss.sum())} of "
              f"{zero.size} NaN; clean recordings bit-identical to the batch without them")
        # what the library does (DESIGN.md §3.8): the NaN sample's own loss is NaN, and the samples whose mel frames
        # read it score finite values (the conditioning's ReLU and the loss's maxima drop a NaN operand); 0 / 0 makes
        # every sample of the silent recording NaN
        assert np.array_equal(np.flatnonzero(nan_loss), [bad_at]) and zero_loss.all()
    finally:
        an.close()
        eng.close()


@pytest.fixture(scope="module")
def lib():
    return cabi.load()
