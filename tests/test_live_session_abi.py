"""Host-side pieces of live sessions (wrnn_live_*), checked without a device: the poll's delivery by ticket-tagged
progress words (wrnn_debug_live_session_deliver, on a host buffer laid out as the session's pinned one), CTA 0's
per-slot decisions at admission boundaries (wrnn_debug_live_session_slot, the functions the kernel runs), the tags and
step indices at their wrap points, and the refusals that need no handle."""
import ctypes
import sys

import numpy as np
import pytest

from wavernn_b200 import cabi

HOP = 275
RETIRED = 1 << 31
PERIOD, DRAIN, ADMIT_LIMIT, MAX_STEPS = 64, 4, 1 << 27, 1 << 27


@pytest.fixture(scope="module")
def lib():
    if not cabi.is_built():
        import __graft_entry__ as g
        g.build()
    return cabi.load()


def _word(lib, ticket, count, retired=False):
    return (lib.wrnn_debug_live_tag(ticket) << 32) | (RETIRED if retired else 0) | count


def _deliver(lib, x, progress, tickets, Ts, delivered, wav, mu_law=False, n_classes=30):
    progress = np.ascontiguousarray(progress, dtype=np.uint64)
    tickets = np.ascontiguousarray(tickets, dtype=np.int64)
    Ts = np.ascontiguousarray(Ts, dtype=np.int64)
    released = np.zeros(len(Ts), dtype=np.int32)
    rc = lib.wrnn_debug_live_session_deliver(x.ctypes.data, x.shape[1], progress.ctypes.data, len(Ts), tickets.ctypes.data,
                                             Ts.ctypes.data, HOP, int(mu_law), n_classes, delivered.ctypes.data,
                                             released.ctypes.data, wav.ctypes.data)
    assert rc == 0, lib.wrnn_last_error()
    return released


def _epilogue(lib, x, wave_len, mu_law=False, n_classes=30):
    wav = np.full(wave_len, np.nan)
    x = np.ascontiguousarray(x[:wave_len], dtype=np.float32)
    assert lib.wrnn_debug_live_epilogue(x.ctypes.data, wave_len, wave_len, HOP, int(mu_law), n_classes, wav.ctypes.data) == 0
    return wav


@pytest.mark.parametrize("mode,mu_law", [("MOL", False), ("RAW", True)])
def test_delivery_follows_each_tickets_tagged_word(lib, mode, mu_law):
    """Slot 0 holds ticket 7 while its word still carries the previous occupant's (ticket 3, retired, with a count past
    ticket 7's): nothing is delivered until ticket 7's own word appears.  Slot 1's ticket advances and retires; slot 2 is
    free.  Each waveform at the end is the unbatched epilogue over its own samples."""
    n_classes = 30 if mode == "MOL" else 512
    Ts = np.array([30, 21, 21], dtype=np.int64)
    steps = 40 * HOP
    rs = np.random.RandomState(2)
    x = rs.uniform(-1, 1, size=(3, steps)).astype(np.float32)
    if mode == "RAW":
        x = (np.float32(2) * rs.randint(0, n_classes, size=(3, steps)).astype(np.float32) / np.float32(n_classes - 1) - 1).astype(np.float32)
    wave = (Ts - 1) * HOP
    tickets = [7, 5, 0]
    wav = np.full(int(wave[0] + wave[1]), np.nan)
    delivered = np.zeros(3, dtype=np.int64)
    stale = _word(lib, 3, 39 * HOP, retired=True)
    rel = _deliver(lib, x, [stale, _word(lib, 5, 0), 0], tickets, Ts, delivered, wav, mu_law, n_classes)
    assert list(delivered) == [0, 0, 0] and not rel.any() and np.isnan(wav).all()
    history = [delivered.copy()]
    for k in range(1, 200):
        w0 = _word(lib, 7, min(64 * k, int(wave[0]) + HOP))             # the fold may publish past its waveform
        n1 = min(128 * k, int(wave[1]))
        w1 = _word(lib, 5, n1, retired=n1 == wave[1] and k % 2 == 0)
        rel = _deliver(lib, x, [w0, w1, 0], tickets, Ts, delivered, wav, mu_law, n_classes)
        assert np.all(delivered >= history[-1]) and delivered[0] == min(64 * k, wave[0])
        history.append(delivered.copy())
        if rel[1]:
            assert delivered[1] == wave[1]
            tickets[1] = 0                                   # released: the poll forgets the slot
        if delivered[0] == wave[0]:
            break
    assert tickets[1] == 0
    assert np.array_equal(wav[:wave[0]].view(np.int64), _epilogue(lib, x[0], int(wave[0]), mu_law, n_classes).view(np.int64))
    assert np.array_equal(wav[wave[0]:].view(np.int64), _epilogue(lib, x[1], int(wave[1]), mu_law, n_classes).view(np.int64))


def test_delivered_samples_are_never_rewritten_and_cancellation_releases(lib):
    Ts = np.array([25, 22], dtype=np.int64)
    x = np.random.RandomState(1).uniform(-1, 1, size=(2, 24 * HOP)).astype(np.float32)
    wave = (Ts - 1) * HOP
    wav = np.full(int(wave.sum()), np.nan)
    delivered = np.zeros(2, dtype=np.int64)
    _deliver(lib, x, [_word(lib, 1, 128), _word(lib, 2, 640)], [1, 2], Ts, delivered, wav)
    assert list(delivered) == [128, 640]
    wav[:128] = 7.0
    wav[wave[0]:wave[0] + 640] = 9.0
    _deliver(lib, x, [_word(lib, 1, 128), _word(lib, 2, 640)], [1, 2], Ts, delivered, wav)
    assert (wav[:128] == 7.0).all() and (wav[wave[0]:wave[0] + 640] == 9.0).all()
    # ticket 1 cancelled: CTA 0 stops it at a boundary and retires it with the count it reached
    rel = _deliver(lib, x, [_word(lib, 1, 192, retired=True), _word(lib, 2, 704)], [1, 2], Ts, delivered, wav)
    assert list(rel) == [1, 0] and list(delivered) == [192, 704]
    assert (wav[:128] == 7.0).all() and np.array_equal(wav[128:192], x[0, 128:192].astype(np.float64))
    assert np.isnan(wav[192:wave[0]]).all()


def _slot(lib, state, seed, b, req, cancel, req_seed=0, steps=1000):
    st = np.ascontiguousarray(state, dtype=np.int64)
    sd = ctypes.c_uint64(seed)
    words = np.zeros(2, dtype=np.uint64)
    assert lib.wrnn_debug_live_session_slot(st.ctypes.data, ctypes.byref(sd), b, req, cancel, req_seed, steps,
                                            words.ctypes.data) == 0, lib.wrnn_last_error()
    return list(st), sd.value, [int(w) for w in words]


def test_slot_decisions_at_boundaries(lib):
    """Admission at the next boundary, retirement only SES_DRAIN steps after the end, cancellation at the next boundary,
    a request with the occupant's own tag is not a new one."""
    free = [0, 0, 0, 1]                                     # tag, a, e, retired
    s, seed, w = _slot(lib, free, 0, 128, req=5, cancel=0, req_seed=2**40 + 1, steps=1000)
    assert s == [5, 192, 1192, 0] and seed == 2**40 + 1 and w == [0, 5 << 32]
    s2, _, w = _slot(lib, s, seed, 192, req=5, cancel=0)
    assert s2 == s and w == [0, 0]
    s2, _, w = _slot(lib, s, seed, 1152, req=5, cancel=0)        # ends at 1192: retired at the first boundary >= 1196
    assert s2 == s and w == [0, 0]
    s3, _, w = _slot(lib, s, seed, 1280, req=6, cancel=0)        # retired and the next request admitted in one boundary
    assert w[0] == (5 << 32) | RETIRED | 1000 and s3[:4] == [6, 1344, 2344, 0] and w[1] == 6 << 32
    s4, _, w = _slot(lib, s3, 0, 1408, req=6, cancel=6)          # cancelled mid-utterance: ends at the next boundary
    assert s4 == [6, 1344, 1472, 0] and w == [0, 0]
    s5, _, w = _slot(lib, s4, 0, 1536, req=6, cancel=6)
    assert s5[3] == 1 and w[0] == (6 << 32) | RETIRED | 128


def test_step_indices_and_tags_at_their_wrap_points(lib):
    """No admission from SES_ADMIT_LIMIT on, so the last step index of a launch stays near 2^28 (five exchanges per
    step of a 32-bit int stay below 2^31); tags never take the value 0 of a never-used slot, and consecutive tickets differ
    across 2^32."""
    last = ADMIT_LIMIT - PERIOD
    s, _, w = _slot(lib, [0, 0, 0, 1], 0, last, req=9, cancel=0, steps=MAX_STEPS)
    assert w[1] == 9 << 32 and s[2] == last + PERIOD + MAX_STEPS == 1 << 28
    assert 5 * (s[2] + DRAIN + 2 * PERIOD) < 2**31                # the launch's last step, times five exchanges
    s, _, w = _slot(lib, [0, 0, 0, 1], 0, ADMIT_LIMIT, req=9, cancel=0)
    assert w == [0, 0] and s == [0, 0, 0, 1]
    tags = [lib.wrnn_debug_live_tag(t) for t in (1, 2, 2**32 - 1, 2**32, 2**32 + 1, 2**33, 2**40 + 7)]
    assert 0 not in tags
    for t in (2**32 - 2, 2**32 - 1, 2**32, 2**33 - 1):
        assert lib.wrnn_debug_live_tag(t) != lib.wrnn_debug_live_tag(t + 1)
    assert lib.wrnn_debug_live_tag(1) == 1 and lib.wrnn_debug_live_tag(2**32 - 1) == 2**32 - 1


def test_refusals_without_a_device(lib):
    def refused(rc, match):
        msg = lib.wrnn_last_error().decode()
        assert rc == cabi.WRNN_E_INVALID and match in msg, (rc, msg)
    refused(lib.wrnn_live_open(None, 0, 100, 0, None), "1 to 64 slots")
    refused(lib.wrnn_live_open(None, 65, 100, 0, None), "1 to 64 slots")
    refused(lib.wrnn_live_open(None, 4, 20, 0, None), "max_T must be >= 21")
    refused(lib.wrnn_live_open(None, 4, 21, 0, None), "null handle")
    tk = ctypes.c_int64(-1)
    u = cabi.WrnnUtterance(0x1000, 26, 1, 0x1000)
    refused(lib.wrnn_live_submit(None, None, ctypes.byref(tk)), "null utterance or ticket")
    refused(lib.wrnn_live_submit(None, ctypes.byref(u), None), "null utterance or ticket")
    refused(lib.wrnn_live_submit(None, ctypes.byref(cabi.WrnnUtterance(None, 26, 1, 0x1000)), ctypes.byref(tk)), "mel and wav")
    refused(lib.wrnn_live_submit(None, ctypes.byref(cabi.WrnnUtterance(0x1000, 20, 1, 0x1000)), ctypes.byref(tk)), "T must be >= 21")
    refused(lib.wrnn_live_submit(None, ctypes.byref(u), ctypes.byref(tk)), "null handle")
    assert tk.value == -1
    refused(lib.wrnn_live_cancel(None, 1), "null handle")
    out = (cabi.WrnnLiveTicket * 8)()
    n = ctypes.c_int32(-1)
    refused(lib.wrnn_live_poll(None, 0, None, 8, ctypes.byref(n)), "null out or n_out")
    refused(lib.wrnn_live_poll(None, 0, out, 8, None), "null out or n_out")
    refused(lib.wrnn_live_poll(None, 0, out, 8, ctypes.byref(n)), "null handle")
    refused(lib.wrnn_live_close(None), "null handle")
    x, wav, d = np.zeros((1, 30 * HOP), np.float32), np.zeros(30 * HOP), np.zeros(1, np.int64)
    T, tks, p, r = np.array([32], np.int64), np.array([1], np.int64), np.zeros(1, np.uint64), np.zeros(1, np.int32)
    hook = lib.wrnn_debug_live_session_deliver
    assert hook(x.ctypes.data, 30 * HOP, p.ctypes.data, 1, tks.ctypes.data, T.ctypes.data, HOP, 0, 30, d.ctypes.data,
                r.ctypes.data, wav.ctypes.data) == cabi.WRNN_E_INVALID             # longer than the slot's row
    assert hook(x.ctypes.data, 30 * HOP, p.ctypes.data, 65, tks.ctypes.data, T.ctypes.data, HOP, 0, 30, d.ctypes.data,
                r.ctypes.data, wav.ctypes.data) == cabi.WRNN_E_INVALID


if __name__ == "__main__":
    sys.exit(pytest.main([__file__, "-v", "-s"]))
