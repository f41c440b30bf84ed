"""Host-side pieces of live batch vocoding (wrnn_vocode_many_live_start / _poll), checked without a device: each poll's
per-utterance delivery (through the wrnn_debug_live_many_deliver hook, on a host buffer laid out as the job's pinned
one) against wrnn_debug_live_epilogue on utterances of different lengths, and the refusals that need no handle."""
import ctypes
import sys

import numpy as np
import pytest

from wavernn_b200 import cabi

HOP = 275
FAKE = 0x1000                      # the refusals below come before any pointer is read


@pytest.fixture(scope="module")
def lib():
    if not cabi.is_built():
        import __graft_entry__ as g
        g.build()
    return cabi.load()


def _epilogue(lib, x, wave_len, mu_law, n_classes):
    wav = np.full(wave_len, np.nan)
    x = np.ascontiguousarray(x, dtype=np.float32)
    assert lib.wrnn_debug_live_epilogue(x.ctypes.data, wave_len, wave_len, HOP, int(mu_law), n_classes, wav.ctypes.data) == 0
    return wav


def _deliver(lib, x, progress, Ts, mu_law, n_classes, delivered, wav):
    progress = np.ascontiguousarray(progress, dtype=np.uint64)
    Ts = np.ascontiguousarray(Ts, dtype=np.int64)
    rc = lib.wrnn_debug_live_many_deliver(x.ctypes.data, x.shape[1], progress.ctypes.data, len(Ts), Ts.ctypes.data, HOP,
                                          int(mu_law), n_classes, delivered.ctypes.data, wav.ctypes.data)
    assert rc == 0, lib.wrnn_last_error()


@pytest.mark.parametrize("mode,mu_law", [("MOL", False), ("RAW", False), ("RAW", True)])
def test_poll_delivers_each_utterance_by_its_own_progress(lib, mode, mu_law):
    """Utterances of 21, 30, 57 and 44 frames in one job of max T * hop steps per fold.  A sequence of published progress
    words, each fold advancing by 64 steps at its own pace (and past its own waveform's end, as the kernel's folds do),
    is delivered poll by poll: each utterance receives min(progress, wave_len) leading samples, never loses any, and its
    waveform at the end is wrnn_debug_live_epilogue's over its own fold."""
    n_classes = 30 if mode == "MOL" else 512
    Ts = np.array([21, 30, 57, 44], dtype=np.int64)
    steps = int(Ts.max()) * HOP
    wave = (Ts - 1) * HOP
    rs = np.random.RandomState(3)
    f = np.float32
    if mode == "RAW":
        x = (f(2) * rs.randint(0, n_classes, size=(len(Ts), steps)).astype(f) / (f(n_classes) - f(1)) - f(1)).astype(f)
    else:
        x = rs.uniform(-1, 1, size=(len(Ts), steps)).astype(f)
    x[1, 5] = f(-0.0)                                      # 0.0 + y: a -0.0 sample becomes +0.0
    wav = np.full(int(wave.sum()), np.nan)
    off = np.concatenate([[0], np.cumsum(wave)])
    delivered = np.zeros(len(Ts), dtype=np.int64)
    pace = np.array([3, 1, 2, 5])                           # periods of 64 steps per poll
    progress = np.zeros(len(Ts), dtype=np.int64)
    history = []
    while True:
        before = delivered.copy()
        progress = np.minimum(progress + 64 * pace, steps)
        _deliver(lib, x, progress, Ts, mu_law, n_classes, delivered, wav)
        assert np.array_equal(delivered, np.minimum(progress, wave)) and np.all(delivered >= before)
        for i in range(len(Ts)):                            # nothing past what this poll reported is written
            assert np.isnan(wav[off[i] + delivered[i]:off[i + 1]]).all()
        history.append(delivered.copy())
        if np.all(progress == steps):
            break
    # utterance 0 (the shortest) is complete while others are not
    assert any(h[0] == wave[0] and np.any(h < wave) for h in history)
    for i in range(len(Ts)):
        want = _epilogue(lib, x[i], int(wave[i]), mu_law, n_classes)
        assert np.array_equal(wav[off[i]:off[i + 1]].view(np.int64), want.view(np.int64)), i
    if not mu_law:
        assert wav[off[1] + 5] == 0 and not np.signbit(wav[off[1] + 5])


def test_poll_does_not_rewrite_delivered_samples(lib):
    """A second delivery at the same progress writes nothing, and one at a later progress only the new samples."""
    Ts = np.array([25, 22], dtype=np.int64)
    steps = 25 * HOP
    x = np.random.RandomState(1).uniform(-1, 1, size=(2, steps)).astype(np.float32)
    wav = np.full(int(((Ts - 1) * HOP).sum()), np.nan)
    delivered = np.zeros(2, dtype=np.int64)
    _deliver(lib, x, [128, 640], Ts, False, 30, delivered, wav)
    assert list(delivered) == [128, 640]
    w0 = (Ts[0] - 1) * HOP
    wav[:128] = 7.0                                        # a caller's marks on delivered samples stay untouched
    wav[w0:w0 + 640] = 9.0
    _deliver(lib, x, [128, 640], Ts, False, 30, delivered, wav)
    assert (wav[:128] == 7.0).all() and (wav[w0:w0 + 640] == 9.0).all() and np.isnan(wav[128:w0]).all()
    _deliver(lib, x, [192, 640], Ts, False, 30, delivered, wav)
    assert (wav[:128] == 7.0).all() and np.array_equal(wav[128:192], x[0, 128:192].astype(np.float64))
    assert list(delivered) == [192, 640]


def _batch(n=3, batched=0, T=26, mel=FAKE, wav=FAKE, at=None):
    utts = [(FAKE, 26, 7 + i, FAKE) for i in range(n)]
    if at is not None:
        utts[at] = (mel, T, 7, wav)
    return cabi.vocode_batch(utts, batched=batched, target=2200, overlap=220)


def test_live_many_refusals_without_a_device(lib):
    """Every refusal that needs no handle comes before the handle check, with its message."""
    def refused(bk, match):
        b = bk[0] if bk is not None else None
        rc = lib.wrnn_vocode_many_live_start(None, ctypes.byref(b) if b is not None else None, None)
        msg = lib.wrnn_last_error().decode()
        assert rc == cabi.WRNN_E_INVALID and match in msg, (rc, msg)
        return msg
    refused(None, "null batch")
    assert "last step" in refused(_batch(batched=1), "unbatched")
    refused(_batch(n=0), "1 to 64 utterances")
    assert "second tile" in refused(_batch(n=65), "1 to 64 utterances")
    b, keep = _batch()
    b.utts = None
    refused((b, keep), "utts is required")
    refused(_batch(at=1, mel=0), "utterance 1: mel and wav are required")
    refused(_batch(at=2, wav=0), "utterance 2: mel and wav are required")
    refused(_batch(at=2, T=20), "utterance 2: T must be >= 21")
    refused(_batch(n=64), "null handle")
    n = np.full(4, -1, dtype=np.int64)
    assert lib.wrnn_vocode_many_live_poll(None, 0, n.ctypes.data) == cabi.WRNN_E_INVALID and (n == -1).all()
    x, wav, d = np.zeros((1, 30 * HOP), np.float32), np.zeros(30 * HOP), np.zeros(1, np.int64)
    T = np.array([30], np.int64)
    p = np.zeros(1, np.uint64)
    hook = lib.wrnn_debug_live_many_deliver
    assert hook(x.ctypes.data, 30 * HOP, p.ctypes.data, 65, T.ctypes.data, HOP, 0, 30, d.ctypes.data, wav.ctypes.data) == cabi.WRNN_E_INVALID
    T[0] = 31                                             # longer than the fold
    assert hook(x.ctypes.data, 30 * HOP, p.ctypes.data, 1, T.ctypes.data, HOP, 0, 30, d.ctypes.data, wav.ctypes.data) == cabi.WRNN_E_INVALID


if __name__ == "__main__":
    sys.exit(pytest.main([__file__, "-v", "-s"]))
