"""Live batch vocoding (wrnn_vocode_many_live_start / _poll) on the device: every waveform delivered while the persistent
kernel runs is bit-identical to wrnn_vocode_many_host's on the same batch (and so to its own unbatched wrnn_vocode_host),
at tile sizes that run the small and the BIG live kernels; each utterance arrives progressively, a short one completes
before the job ends, the handle refuses other work while the job is in flight, and what cannot run live is refused."""
import ctypes

import numpy as np
import pytest

import helpers
from wavernn_b200 import cabi

pytestmark = pytest.mark.gpu

HOP = 275


@pytest.fixture(scope="module")
def lib():
    if not cabi.is_built():
        import __graft_entry__ as g
        g.build()
    return cabi.load()


def _engine(model, precision="fp16", engine="tcgen05"):
    eng = cabi.Engine(model.hot_state(), n_classes=model.n_classes, mode=model.mode, precision=precision, engine=engine)
    eng.attach_upsampler(model.state_dict())
    return eng


def _mels(Ts, seed):
    return [np.ascontiguousarray(helpers.make_mel(T, seed=seed + i)[0].numpy()) for i, T in enumerate(Ts)]


def _live(eng, mels, seeds, **kw):
    """The waveforms vocode_many_live yields, concatenated per utterance, and the number of slices of each."""
    parts = [[] for _ in mels]
    for i, part in eng.vocode_many_live(mels, seeds, **kw):
        parts[i].append(part.copy())
    return [np.concatenate(p) if p else np.empty(0) for p in parts], [len(p) for p in parts]


def _same(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.int64), b.view(np.int64))


@pytest.mark.parametrize("mode,precision,mu_law", [("MOL", "fp16", False), ("MOL", "bf16", False), ("RAW", "fp16", True),
                                                   ("RAW", "bf16", False)])
def test_live_many_equals_vocode_many_host(lib, mode, precision, mu_law):
    m = helpers.make_model(0, mode)
    eng = _engine(m, precision)
    Ts, seeds = [40, 26, 61, 33], [1234, 7, 99, 2**40 + 3]
    mels = _mels(Ts, 20)
    got, n_parts = _live(eng, mels, seeds, mu_law=mu_law)
    assert eng.name.startswith("tcgen05")
    want = eng.vocode_many_host(mels, seeds, batched=False, mu_law=mu_law)
    print(f"{mode} {precision} mu_law={mu_law}: slices per utterance {n_parts}")
    for i, mel in enumerate(mels):
        assert _same(got[i], want[i]), i
        assert _same(got[i], eng.vocode_host(mel, batched=False, mu_law=mu_law, philox_seed=seeds[i])), i


@pytest.mark.parametrize("n", [1, 24, 25, 64])
def test_live_many_tile_sizes(lib, n):
    """1 and 24 utterances run the small live kernel, 25 and 64 the BIG one."""
    m = helpers.make_model(0, "MOL")
    eng = _engine(m)
    Ts = [21 + (7 * i) % 10 for i in range(n)]
    seeds = [5 + 3 * i for i in range(n)]
    mels = _mels(Ts, 100)
    got, _ = _live(eng, mels, seeds)
    want = eng.vocode_many_host(mels, seeds, batched=False)
    for i in range(n):
        assert _same(got[i], want[i]), i


def test_live_many_on_the_checkpoint(lib):
    m = helpers.make_model(0, "MOL")
    m.load_state_dict(helpers.pretrained_state_dict())
    eng = _engine(m)
    mels = list(helpers.tacotron_mels()[:4])
    seeds = [77, 78, 79, 80]
    got, _ = _live(eng, mels, seeds)
    want = eng.vocode_many_host(mels, seeds, batched=False)
    for i in range(4):
        assert _same(got[i], want[i]), i
        assert np.abs(got[i]).max() > 1e-3                # a waveform, not silence


def _start(lib, eng, mels, wavs, seeds, mu_law=False):
    b, keep = cabi.vocode_batch([(x.ctypes.data, x.shape[1], s, w.ctypes.data) for x, s, w in zip(mels, seeds, wavs)],
                                batched=False, mu_law=mu_law)
    return lib.wrnn_vocode_many_live_start(eng._h, ctypes.byref(b), None)


def _drain(lib, eng, wavs):
    """Polls to the end; per poll: return code, n_ready copy, and per utterance (prev, copy of the newly final slice)."""
    n = np.zeros(len(wavs), dtype=np.int64)
    prev, polls = n.copy(), []
    while True:
        rc = lib.wrnn_vocode_many_live_poll(eng._h, 1000, n.ctypes.data)
        polls.append((rc, n.copy(), [(int(prev[i]), wavs[i][prev[i]:n[i]].copy()) for i in range(len(wavs))]))
        prev = np.maximum(prev, n)
        if rc != 1:
            return polls


def test_live_many_delivery_is_progressive_and_final(lib):
    m = helpers.make_model(0, "MOL")
    eng = _engine(m)
    Ts, seeds = [21, 400, 150], [5, 6, 7]
    mels = _mels(Ts, 40)
    wave = [(T - 1) * HOP for T in Ts]
    wavs = [np.full(w, np.nan) for w in wave]
    assert _start(lib, eng, mels, wavs, seeds) == 0
    polls = _drain(lib, eng, wavs)
    assert polls[-1][0] == 0 and list(polls[-1][1]) == wave
    ns = np.array([p[1] for p in polls])
    assert np.all(np.diff(ns, axis=0) >= 0), "n_ready decreased"
    partial = [p for p in polls if p[0] == 1 and 0 < p[1][1] < wave[1]]
    short_done = [p for p in polls if p[0] == 1 and p[1][0] == wave[0]]
    print(f"{len(polls)} polls, {len(partial)} returned 1 with 0 < n_ready[1] < {wave[1]}, "
          f"{len(short_done)} returned 1 with the short utterance complete")
    assert partial and short_done
    for _, n, parts in polls:              # what each poll delivered is what the waveforms hold at the end
        for i, (prev, part) in enumerate(parts):
            assert np.array_equal(part.view(np.int64), wavs[i][prev:n[i]].view(np.int64))
    want = eng.vocode_many_host(mels, seeds, batched=False)
    for i in range(3):
        assert _same(wavs[i], want[i]), i


def test_handle_is_busy_during_a_live_batch(lib):
    m = helpers.make_model(0, "RAW")
    eng = _engine(m, "bf16")
    mels = _mels([400, 300], 60)
    seeds = [8, 9]
    short = helpers.make_mel(26, seed=2)[0].numpy()
    before = eng.vocode_host(short, batched=False, mu_law=True, philox_seed=3)
    before_many = eng.vocode_many_host([short, short], [3, 4], batched=False)
    wavs = [np.full((x.shape[1] - 1) * HOP, np.nan) for x in mels]
    assert _start(lib, eng, mels, wavs, seeds, mu_law=True) == 0

    def busy(fn, *a, **k):
        with pytest.raises(cabi.EngineError, match="wrnn_vocode_many_live_poll until") as e:
            fn(*a, **k)
        assert e.value.code == cabi.WRNN_E_BUSY
    busy(eng.vocode_host, short, batched=False, philox_seed=3)
    busy(eng.vocode_many_host, [short], [3], batched=False)
    busy(eng.score_many_host, [short], [np.zeros(25 * HOP, np.float32)])
    busy(eng.check)
    busy(lambda: list(eng.vocode_live(short, philox_seed=1)))
    busy(lambda: list(eng.vocode_many_live([short], [1])))
    # the single job's poll does not serve this job and leaves it alone
    one = ctypes.c_int64(-1)
    assert lib.wrnn_vocode_live_poll(eng._h, 0, ctypes.byref(one)) == cabi.WRNN_E_INVALID and one.value == -1
    assert b"wrnn_vocode_many_live_poll" in lib.wrnn_last_error()
    polls = _drain(lib, eng, wavs)
    assert polls[-1][0] == 0 and list(polls[-1][1]) == [w.size for w in wavs]
    n = np.full(2, -1, dtype=np.int64)
    assert lib.wrnn_vocode_many_live_poll(eng._h, 0, n.ctypes.data) == cabi.WRNN_E_INVALID and (n == -1).all()
    want = eng.vocode_many_host(mels, seeds, batched=False, mu_law=True)
    for i in range(2):
        assert _same(wavs[i], want[i])
    assert np.array_equal(eng.vocode_host(short, batched=False, mu_law=True, philox_seed=3), before)
    for a, b in zip(eng.vocode_many_host([short, short], [3, 4], batched=False), before_many):
        assert _same(a, b)

    # and the other way: during a single live job, the batch poll refuses without touching it
    wav1 = np.full((mels[0].shape[1] - 1) * HOP, np.nan)
    job = cabi.WrnnVocodeJob(mels[0].ctypes.data, mels[0].shape[1], 0, 0, 0, 0, 8, wav1.ctypes.data)
    assert lib.wrnn_vocode_live_start(eng._h, ctypes.byref(job), None) == 0
    assert _start(lib, eng, mels, wavs, seeds) == cabi.WRNN_E_BUSY
    n = np.full(2, -1, dtype=np.int64)
    assert lib.wrnn_vocode_many_live_poll(eng._h, 0, n.ctypes.data) == cabi.WRNN_E_INVALID and (n == -1).all()
    assert b"wrnn_vocode_live_poll" in lib.wrnn_last_error()
    rc = 1
    while rc == 1:
        rc = lib.wrnn_vocode_live_poll(eng._h, 1000, ctypes.byref(one))
    assert rc == 0 and one.value == wav1.size
    assert _same(wav1, eng.vocode_host(mels[0], batched=False, philox_seed=8))


def test_destroy_waits_for_a_live_batch(lib):
    m = helpers.make_model(0, "MOL")
    eng = _engine(m)
    mels = _mels([100, 60, 80], 70)
    wavs = [np.full((x.shape[1] - 1) * HOP, np.nan) for x in mels]
    assert _start(lib, eng, mels, wavs, [2, 3, 4]) == 0
    eng.close()
    eng = _engine(m)                                     # the device is usable after the handle that ran the job is gone
    assert all(np.isfinite(w).all() for w in eng.vocode_many_host(mels, [2, 3, 4], batched=False))


def test_refusals_leave_the_handle_usable(lib):
    m = helpers.make_model(0, "MOL")
    mels = _mels([26, 30], 3)

    def refused(eng, match, ms=mels):
        with pytest.raises(cabi.EngineError, match=match) as e:
            list(eng.vocode_many_live(ms, list(range(len(ms)))))
        assert e.value.code == cabi.WRNN_E_INVALID
        assert all(np.isfinite(w).all() for w in eng.vocode_many_host(mels, [0, 1], batched=False))
    refused(_engine(m, "fp16", "stream"), "stream engine's cluster form takes about 66 us per step")
    refused(_engine(m, "fp32", "auto"), "SIMT engine's step has not been timed")
    refused(_engine(m, "bf16", "simt"), "SIMT engine")
    bare = cabi.Engine(m.hot_state())
    with pytest.raises(cabi.EngineError, match="no upsampler attached"):
        list(bare.vocode_many_live(mels, [0, 1]))
    eng = _engine(m)
    first = eng.vocode_many_host(mels, [0, 1], batched=False)
    refused(eng, "1 to 64 utterances", [mels[0]] * 65)
    b, keep = cabi.vocode_batch([(x.ctypes.data, x.shape[1], i, 1) for i, x in enumerate(mels)], batched=True,
                                target=2200, overlap=220)
    assert lib.wrnn_vocode_many_live_start(eng._h, ctypes.byref(b), None) == cabi.WRNN_E_INVALID
    assert b"a batched job's folds all finish at its last step" in lib.wrnn_last_error()
    with pytest.raises(cabi.EngineError, match="utterance 1: T must be >= 21"):
        list(eng.vocode_many_live([mels[0], mels[1][:, :20]], [0, 1]))
    got, _ = _live(eng, mels, [0, 1])
    for a, b_ in zip(got, first):
        assert _same(a, b_)
