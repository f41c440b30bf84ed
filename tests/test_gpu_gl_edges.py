"""Griffin-Lim (wrnn_griffinlim_many) at its edges, on the GPU.

  1. The kernels on every cell of tests/mel_edges.py's grid and every mel of tests/gl_edges.py, in one guarded batch
     per cell at n_iter 0, 1 and 2: against the oracle under gl_edges.local_steps at gl_edges.LOCAL_TOL, and against
     the host run of the same code (reported, not asserted: the device FFT stages are contracted into FMAs).  The mels
     sit in one buffer and the waveforms in another, each between GUARD sentinel words (a NaN payload): a read outside
     a mel or a waveform turns samples NaN, a stray write breaks a sentinel, and the guarded batch equals an unguarded
     one bit for bit.  The batch equals each mel run alone, and the host entry the device entry.
  2. Launch batches: at n_fft = 4096 a call splits into runs of whole utterances of at most GL_CHUNK_BYTES of scratch.
     A batch of tiled Tacotron mels that spans five launch batches (an utterance ending exactly at the cap, one crossing
     it by one frame, one longer than the cap, short utterances on both sides) equals each utterance run alone, the
     host entry and the reversed batch; a NaN mel in the second launch batch leaves every other utterance bit-identical.
  3. Two streams sharing one analysis object equal sequential calls; 2,000 short utterances in one call, in two
     orders, equal each other and each utterance run alone.
Run on a GPU: pytest -m gpu -s tests/test_gpu_gl_edges.py"""
import numpy as np
import pytest
import torch

import gl_edges as E
import helpers
from test_gl_abi import host_gl
from wavernn_b200 import cabi

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
SENTINEL = 0x7FA5A5A5            # a NaN payload no arithmetic produces
GUARD = 64                       # sentinel words on each side of each mel and each waveform
GL_CHUNK_BYTES = 1 << 30         # wrnn_mel.cu: scratch per launch batch


def bits(a):
    return np.ascontiguousarray(a).view(np.int32)


def gl_device(an, mels, seeds, n_iter, stream=None):
    """wrnn_griffinlim_many on device copies of mels, each in a tensor of its own; returns the host waveforms."""
    st = stream or torch.cuda.current_stream(DEV)
    with torch.cuda.stream(st):
        dm = [torch.as_tensor(np.ascontiguousarray(m, dtype=np.float32)).to(DEV) for m in mels]
        dw = [torch.full((an.samples(m.shape[1]),), float("nan"), device=DEV) for m in mels]
        an.griffinlim_many(mels=[m.data_ptr() for m in dm], Ts=[m.shape[1] for m in mels], seeds=seeds,
                           wavs=[w.data_ptr() for w in dw], n_iter=n_iter, stream=st.cuda_stream)
    if stream is not None:
        return dw, dm
    torch.cuda.synchronize(DEV)
    return [w.cpu().numpy() for w in dw]


def gl_guarded(an, mels, seeds, n_iter):
    """One wrnn_griffinlim_many batch with the mels in one int32 buffer and the waveforms in another, each between
    GUARD sentinel words: (host waveforms, whether every sentinel of both buffers survived)."""
    Ts = [m.shape[1] for m in mels]
    moffs = np.cumsum([0] + [m.size + GUARD for m in mels])
    hm = np.full(int(moffs[-1]) + GUARD, SENTINEL, np.int32)
    for o, m in zip(moffs, mels):
        hm[o + GUARD:o + GUARD + m.size] = bits(np.ascontiguousarray(m, dtype=np.float32)).reshape(-1)
    dm = torch.from_numpy(hm).to(DEV)
    ns = [an.samples(T) for T in Ts]
    woffs = np.cumsum([0] + [n + GUARD for n in ns])
    dw = torch.full((int(woffs[-1]) + GUARD,), SENTINEL, dtype=torch.int32, device=DEV)
    an.griffinlim_many(mels=[dm.data_ptr() + 4 * int(o + GUARD) for o in moffs[:-1]], Ts=Ts, seeds=seeds,
                       wavs=[dw.data_ptr() + 4 * int(o + GUARD) for o in woffs[:-1]], n_iter=n_iter,
                       stream=torch.cuda.current_stream(DEV).cuda_stream)
    torch.cuda.synchronize(DEV)
    h = dw.cpu().numpy()
    wavs = [h[o + GUARD:o + GUARD + n].view(np.float32).copy() for o, n in zip(woffs, ns)]
    keep = np.ones(h.size, bool)
    for o, n in zip(woffs, ns):
        keep[o + GUARD:o + GUARD + n] = False
    intact = bool((h[keep] == SENTINEL).all()) and np.array_equal(dm.cpu().numpy(), hm)
    return wavs, intact


# ---- 1. the grid -----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def grid_worst():
    return {}


@pytest.mark.parametrize("name", list(E.GRID))
def test_kernels_on_the_grid(lib, grid_worst, name):
    c = E.cfg(name)
    an = cabi.MelAnalysis(**c)
    try:
        ms = E.mels(c)
        names, mels = list(ms), list(ms.values())
        seeds = [E.SEED] * len(mels)
        worst, vs_host, moved = {}, {}, 0
        for n_iter in (0, 1, 2):
            guarded, intact = gl_guarded(an, mels, seeds, n_iter)
            assert intact, (n_iter, "a write outside a waveform or a mel")
            plain = gl_device(an, mels, seeds, n_iter)
            for k, mel, g, u in zip(names, mels, guarded, plain):
                assert np.array_equal(bits(g), bits(u)), (k, n_iter, "guarded != unguarded")
                assert np.isfinite(g).all(), (k, n_iter, "a read outside a mel or a waveform")
                d = float(E.local_steps(g, E.oracle(mel, n_iter, **c), c).max())
                worst[n_iter] = max(worst.get(n_iter, 0.0), d)
                host, _ = host_gl(lib, mel, E.SEED, n_iter, **c)
                vs_host[n_iter] = max(vs_host.get(n_iter, 0.0), float(E.local_steps(g, host, c).max()))
                moved += int((bits(g) != bits(host)).sum())
                assert d <= E.LOCAL_TOL[n_iter], (k, n_iter, d)
        for k, mel, g in zip(names, mels, plain):
            assert np.array_equal(bits(gl_device(an, [mel], [E.SEED], 2)[0]), bits(g)), (k, "batch != alone")
        assert all(np.array_equal(bits(a), bits(b)) for a, b in zip(an.griffinlim_many_host(mels, 2, seeds), plain))
        grid_worst[name] = worst
        n_out = sum(an.samples(m.shape[1]) for m in mels)
        print(f"{name}: device vs oracle, local float32 steps at n_iter 0/1/2: "
              + " / ".join(f"{worst[n]:.1f}" for n in (0, 1, 2)) + "; vs the host run "
              + " / ".join(f"{vs_host[n]:.1f}" for n in (0, 1, 2))
              + f" ({moved} of {3 * n_out} samples differ); guards and sentinels intact")
    finally:
        an.close()


def test_grid_maximum(grid_worst):
    if len(grid_worst) < len(E.GRID):
        pytest.skip("the grid did not run whole")
    for n in (0, 1, 2):
        name = max(grid_worst, key=lambda k: grid_worst[k][n])
        print(f"n_iter {n}: device vs oracle over the grid {grid_worst[name][n]:.1f} local float32 steps (at {name}); "
              f"LOCAL_TOL {E.LOCAL_TOL[n]}")
        assert grid_worst[name][n] <= E.LOCAL_TOL[n]


# ---- 2. launch batches -----------------------------------------------------------------------------------------------------
def gl_frame_bytes(n_fft):
    """wrnn_mel.cu's scratch per frame: S (float32) and the previous rebuilt bins (complex64), each rounded up to 256
    bytes, and the float64 frame."""
    nb = n_fft // 2 + 1
    return ((nb * 4 + 255) & ~255) + ((nb * 8 + 255) & ~255) + n_fft * 8


def launch_batches(Ts, n_fft):
    """wrnn_mel.cu's split of a call into launch batches: runs of whole utterances of at most cap frames, an utterance
    that would take its run past the cap starting the next (so one longer than the cap runs alone)."""
    cap = max(1, GL_CHUNK_BYTES // gl_frame_bytes(n_fft))
    first, f0 = [0], np.cumsum([0] + list(Ts))
    for i in range(len(Ts)):
        if i > first[-1] and f0[i + 1] - f0[first[-1]] > cap:
            first.append(i)
    first.append(len(Ts))
    return cap, [list(range(a, b)) for a, b in zip(first[:-1], first[1:])]


def tiled_mel(T, start):
    """T frames of the 16 Tacotron mels laid end to end, from frame `start`."""
    taco = np.concatenate(helpers.tacotron_mels(), axis=1)
    reps = (start + T) // taco.shape[1] + 1
    return np.ascontiguousarray(np.tile(taco, (1, reps))[:, start:start + T])


def test_launch_batches():
    c = E.cfg("sr44k")                               # n_fft 4096: the smallest cap, 18,558 frames
    an = cabi.MelAnalysis(**c)
    try:
        cap = GL_CHUNK_BYTES // gl_frame_bytes(c["n_fft"])
        assert cap == 18558
        T0 = E.shortest(c)
        # short | ends exactly at the cap || short || crosses the cap by one || longer than the cap || short, shortest
        Ts = [300, cap - 300, 200, cap - 200 + 1, cap + 1, 150, T0]
        _, batches = launch_batches(Ts, c["n_fft"])
        f0 = np.cumsum([0] + Ts)
        print(f"cap {cap} frames; launch batches (utterances, frames): "
              + " | ".join(f"{b} {int(f0[b[-1] + 1] - f0[b[0]])}" for b in batches))
        assert batches == [[0, 1], [2], [3], [4], [5, 6]]
        assert f0[2] - f0[0] == cap                                   # ends exactly at the cap
        assert f0[4] - f0[2] == cap + 1                               # crosses it by one frame
        assert Ts[4] > cap                                            # alone
        mels = [tiled_mel(T, 997 * i) for i, T in enumerate(Ts)]
        seeds = [11 + i for i in range(len(Ts))]
        batch = gl_device(an, mels, seeds, 2)
        for i, (m, w) in enumerate(zip(mels, batch)):
            assert w.shape == (an.samples(Ts[i]),) and np.isfinite(w).all(), i
            assert np.array_equal(bits(gl_device(an, [m], [seeds[i]], 2)[0]), bits(w)), (i, "batch != alone")
        assert all(np.array_equal(bits(a), bits(b)) for a, b in zip(an.griffinlim_many_host(mels, 2, seeds), batch))
        rev = gl_device(an, mels[::-1], seeds[::-1], 2)[::-1]
        assert all(np.array_equal(bits(a), bits(b)) for a, b in zip(rev, batch)), "reversed batch"
        bad = mels[2].copy()
        bad[40, 100] = np.nan
        poisoned = gl_device(an, mels[:2] + [bad] + mels[3:], seeds, 2)
        assert np.isnan(poisoned[2]).any()
        assert all(np.array_equal(bits(poisoned[i]), bits(batch[i])) for i in range(len(Ts)) if i != 2)
        print(f"{len(Ts)} utterances, {int(f0[-1])} frames in {len(batches)} launch batches: each alone, the host "
              "entry and the reversed batch bit-identical; a NaN mel in the second launch batch confined to itself")
    finally:
        an.close()


# ---- 3. streams and many utterances -----------------------------------------------------------------------------------------
def test_two_streams_share_one_analysis():
    an = cabi.MelAnalysis()
    try:
        taco = helpers.tacotron_mels()
        a, b = taco[:8], taco[8:]
        want_a, want_b = gl_device(an, a, list(range(8)), 3), gl_device(an, b, list(range(8, 16)), 3)
        s1, s2 = torch.cuda.Stream(DEV), torch.cuda.Stream(DEV)
        torch.cuda.synchronize(DEV)
        for _ in range(2):
            da, ma = gl_device(an, a, list(range(8)), 3, stream=s1)
            db, mb = gl_device(an, b, list(range(8, 16)), 3, stream=s2)
            torch.cuda.synchronize(DEV)
            assert all(np.array_equal(bits(w.cpu().numpy()), bits(v)) for w, v in zip(da, want_a))
            assert all(np.array_equal(bits(w.cpu().numpy()), bits(v)) for w, v in zip(db, want_b))
    finally:
        an.close()


def test_two_thousand_short_utterances():
    c = E.cfg("default")
    an = cabi.MelAnalysis(**c)
    try:
        rs = np.random.RandomState(3)
        T0 = E.shortest(c)
        Ts = [T0 + int(rs.randint(0, 12)) if i % 4 else T0 for i in range(2000)]
        mels = [tiled_mel(T, int(rs.randint(0, 5000))) for T in Ts]
        seeds = [int(s) for s in rs.randint(0, 2 ** 62, len(Ts), dtype=np.int64)]
        batch = gl_device(an, mels, seeds, 2)
        perm = rs.permutation(len(mels))
        pb = gl_device(an, [mels[i] for i in perm], [seeds[i] for i in perm], 2)
        for k, i in enumerate(perm):
            assert np.array_equal(bits(pb[k]), bits(batch[i])), i
        for i in range(len(mels)):
            assert np.isfinite(batch[i]).all(), i
            assert np.array_equal(bits(gl_device(an, [mels[i]], [seeds[i]], 2)[0]), bits(batch[i])), i
        print(f"2000 utterances, {sum(Ts)} frames (T = {T0} .. {max(Ts)}): both orders and each alone bit-identical")
    finally:
        an.close()


@pytest.fixture(scope="module")
def lib():
    return cabi.load()
