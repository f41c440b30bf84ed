"""Live unbatched vocoding (wrnn_vocode_live_start / _poll) on the device: the waveform delivered while the persistent
kernel runs is bit-identical to wrnn_vocode_host's, it arrives progressively and is never rewritten, the handle refuses
other work while the job is in flight, and engines other than the persistent one are refused."""
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


def _live(eng, mel, **kw):
    parts = list(eng.vocode_live(mel, **kw))
    return np.concatenate(parts), len(parts)


@pytest.mark.parametrize("mode,precision,mu_law", [("MOL", "fp16", False), ("MOL", "bf16", False), ("RAW", "fp16", True),
                                                   ("RAW", "bf16", False)])
def test_live_equals_vocode_host(lib, mode, precision, mu_law):
    m = helpers.make_model(0, mode)
    eng = _engine(m, precision)
    mel = helpers.make_mel(40, seed=9)[0].numpy()
    got, n_parts = _live(eng, mel, philox_seed=1234, mu_law=mu_law)
    assert eng.name.startswith("tcgen05")
    want = eng.vocode_host(mel, batched=False, mu_law=mu_law, philox_seed=1234)
    print(f"{mode} {precision} mu_law={mu_law}: {got.size} samples in {n_parts} slices")
    assert got.shape == want.shape and np.array_equal(got.view(np.int64), want.view(np.int64))


def test_live_equals_vocode_host_on_the_checkpoint(lib):
    m = helpers.make_model(0, "MOL")
    m.load_state_dict(helpers.pretrained_state_dict())
    eng = _engine(m)
    mel = helpers.tacotron_mels()[0]
    got, _ = _live(eng, mel, philox_seed=77)
    want = eng.vocode_host(mel, batched=False, philox_seed=77)
    assert np.array_equal(got.view(np.int64), want.view(np.int64))
    assert np.abs(got).max() > 1e-3                      # a waveform, not silence


def _start(lib, eng, mel, wav, seed, mu_law=False):
    job = cabi.WrnnVocodeJob(mel.ctypes.data, mel.shape[1], 0, 0, 0, int(mu_law), seed, wav.ctypes.data)
    return lib.wrnn_vocode_live_start(eng._h, ctypes.byref(job), None)


def _drain(lib, eng, wav):
    """Polls to the end; returns the (return code, n_ready, copy of the newly final slice) of every poll."""
    n, prev, polls = ctypes.c_int64(0), 0, []
    while True:
        rc = lib.wrnn_vocode_live_poll(eng._h, 1000, ctypes.byref(n))
        polls.append((rc, n.value, wav[prev:n.value].copy(), prev))
        prev = max(prev, n.value)
        if rc != 1:
            return polls


def test_live_delivery_is_progressive_and_final(lib):
    m = helpers.make_model(0, "MOL")
    eng = _engine(m)
    T = 400
    mel = np.ascontiguousarray(helpers.make_mel(T, seed=4)[0].numpy())
    wave_len = (T - 1) * HOP
    wav = np.full(wave_len, np.nan)
    assert _start(lib, eng, mel, wav, 5) == 0
    polls = _drain(lib, eng, wav)
    assert polls[-1][0] == 0 and polls[-1][1] == wave_len
    ns = [n for _, n, _, _ in polls]
    assert all(b >= a for a, b in zip(ns, ns[1:])), "n_ready decreased"
    partial = [n for rc, n, _, _ in polls if rc == 1 and 0 < n < wave_len]
    print(f"{len(polls)} polls, {len(partial)} returned 1 with 0 < n_ready < {wave_len}; first audio at n_ready = "
          f"{partial[0] if partial else None}")
    assert partial
    for _, n, part, prev in polls:              # what each poll delivered is what the waveform holds at the end
        assert np.array_equal(part.view(np.int64), wav[prev:n].view(np.int64))
    want = eng.vocode_host(mel, batched=False, philox_seed=5)
    assert np.array_equal(wav.view(np.int64), want.view(np.int64))


def test_handle_is_busy_during_a_live_job(lib):
    m = helpers.make_model(0, "RAW")
    eng = _engine(m, "bf16")
    mel = np.ascontiguousarray(helpers.make_mel(400, seed=6)[0].numpy())
    short = helpers.make_mel(26, seed=2)[0].numpy()
    before = eng.vocode_host(short, batched=False, mu_law=True, philox_seed=3)
    wav = np.full(399 * HOP, np.nan)
    assert _start(lib, eng, mel, wav, 8, mu_law=True) == 0

    def busy(fn, *a, **k):
        with pytest.raises(cabi.EngineError, match="live job is in flight") as e:
            fn(*a, **k)
        assert e.value.code == cabi.WRNN_E_BUSY
    busy(eng.vocode_host, short, batched=False, philox_seed=3)
    busy(eng.score_many_host, [short], [np.zeros(25 * HOP, np.float32)])
    wav2 = np.empty_like(wav)
    assert _start(lib, eng, mel, wav2, 8) == cabi.WRNN_E_BUSY
    busy(eng.check)
    polls = _drain(lib, eng, wav)
    assert polls[-1][:2] == (0, wav.size)
    n = ctypes.c_int64(-1)
    assert lib.wrnn_vocode_live_poll(eng._h, 0, ctypes.byref(n)) == cabi.WRNN_E_INVALID and n.value == -1
    assert np.array_equal(eng.vocode_host(short, batched=False, mu_law=True, philox_seed=3), before)
    assert np.array_equal(wav, eng.vocode_host(mel, batched=False, mu_law=True, philox_seed=8))


def test_destroy_waits_for_a_live_job(lib):
    m = helpers.make_model(0, "MOL")
    eng = _engine(m)
    mel = np.ascontiguousarray(helpers.make_mel(100, seed=1)[0].numpy())
    wav = np.full(99 * HOP, np.nan)
    assert _start(lib, eng, mel, wav, 2) == 0
    eng.close()
    eng = _engine(m)                                     # the device is usable after the handle that ran the job is gone
    assert np.isfinite(eng.vocode_host(mel, batched=False, philox_seed=2)).all()


def test_refusals_leave_the_handle_usable(lib):
    m = helpers.make_model(0, "MOL")
    mel = helpers.make_mel(26, seed=3)[0].numpy()

    def refused(eng, match):
        with pytest.raises(cabi.EngineError, match=match) as e:
            list(eng.vocode_live(mel, philox_seed=1))
        assert e.value.code == cabi.WRNN_E_INVALID
        assert np.isfinite(eng.vocode_host(mel, batched=False, philox_seed=1)).all()
    refused(_engine(m, "fp16", "stream"), "stream engine's cluster form takes about 66 us per step")
    refused(_engine(m, "fp32", "auto"), "SIMT engine's step has not been timed")
    refused(_engine(m, "bf16", "simt"), "SIMT engine")
    bare = cabi.Engine(m.hot_state())
    with pytest.raises(cabi.EngineError, match="no upsampler attached"):
        list(bare.vocode_live(mel, philox_seed=1))
    eng = _engine(m)
    first = eng.vocode_host(mel, batched=False, philox_seed=1)
    wav = np.empty(25 * HOP)
    mel_c = np.ascontiguousarray(mel)
    job = cabi.WrnnVocodeJob(mel_c.ctypes.data, 26, 1, 2200, 220, 0, 1, wav.ctypes.data)
    assert lib.wrnn_vocode_live_start(eng._h, ctypes.byref(job), None) == cabi.WRNN_E_INVALID
    assert b"a batched job's folds all finish at its last step" in lib.wrnn_last_error()
    with pytest.raises(cabi.EngineError, match="T must be >= 21"):
        list(eng.vocode_live(mel[:, :20], philox_seed=1))
    assert np.array_equal(_live(eng, mel, philox_seed=1)[0], first)
