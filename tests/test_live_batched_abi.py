"""Host-side pieces of batched live tickets (wrnn_live_submit_batched), checked without a device: one poll's delivery of
a ticket whose folds sit in given slots with given published counts (wrnn_debug_live_batched_deliver, on a host buffer
laid out as the session's pinned one), the relaunch decision for a ticket whose folds a launch served in part
(wrnn_debug_live_batched_relaunch), CTA 0's slot decision for a folded occupant (wrnn_debug_live_session_fold_slot), and
the refusals that need no handle."""
import ctypes
import math
import sys

import numpy as np
import pytest

from oracle import wavernn_oracle as O
from wavernn_b200 import cabi

HOP = 275
RETIRED = 1 << 31


@pytest.fixture(scope="module")
def lib():
    if not cabi.is_built():
        import __graft_entry__ as g
        g.build()
    return cabi.load()


def _word(lib, ticket, count, retired=False):
    return (lib.wrnn_debug_live_tag(ticket) << 32) | (RETIRED if retired else 0) | count


def _samples(rs, shape, mode, n_classes):
    if mode == "MOL":
        return rs.uniform(-1, 1, size=shape).astype(np.float32)
    k = rs.randint(0, n_classes, size=shape).astype(np.float32)
    return (np.float32(2) * k / np.float32(n_classes - 1) - np.float32(1)).astype(np.float32)


class Ticket:
    """One batched ticket of T frames whose fold b is held by slot slots[b] of a session of C slots."""

    def __init__(self, lib, T, target, overlap, slots, C, mode="MOL", mu_law=False, ticket=9, seed=0):
        self.lib, self.T, self.target, self.overlap, self.C = lib, T, target, overlap, C
        self.mode, self.mu_law, self.ticket = mode, mu_law, ticket
        self.n_classes = 30 if mode == "MOL" else 512
        self.n_seg, _ = O.fold_geometry(T * HOP, target, overlap)
        assert len(slots) == self.n_seg
        self.slots = np.ascontiguousarray(slots, dtype=np.int32)
        self.seg_len, self.stride = target + 2 * overlap, target + overlap
        self.wave_len = (T - 1) * HOP
        self.max_steps = self.seg_len + 3 * HOP
        self.x = np.full((C, self.max_steps), np.nan, dtype=np.float32)      # rows of other slots are never read
        self.folds = _samples(np.random.RandomState(seed), (self.n_seg, self.seg_len), mode, self.n_classes)
        self.x[self.slots, :self.seg_len] = self.folds
        self.wav = np.full(self.wave_len, np.nan)
        self.delivered = 0

    def want(self):
        """oracle.epilogue(batched=True).  With mu-law, decode_mu_law is evaluated per sample with the C library's pow, as
        the library's table is (test_vocode_abi.py::test_mu_law_table): numpy's vectorised np.power may differ from it in
        the last bit."""
        y, mu_law = self.folds, self.mu_law
        if mu_law:
            n = self.n_classes
            y = np.vectorize(lambda v: np.sign(v) / (n - 1) * (math.pow(n, abs(v)) - 1))(self.folds.astype(np.float64))
            mu_law = False
        return O.epilogue(y, batched=True, target=self.target, overlap=self.overlap, wave_len=self.wave_len,
                          hop_length=HOP, mode=self.mode, mu_law=mu_law, n_classes=self.n_classes)

    def prefix(self, counts):
        """The longest prefix whose every sample each covering fold has published."""
        ready = self.wave_len
        for b, c in enumerate(counts):
            if c < self.seg_len:
                ready = min(ready, b * self.stride + c)
        return ready

    def deliver(self, words):
        """One poll's delivery with progress[slots[b]] = words[b]; other slots carry another ticket's words."""
        progress = np.array([_word(self.lib, 3, 64, True)] * self.C, dtype=np.uint64)
        progress[self.slots] = np.asarray(words, dtype=np.uint64)
        d = ctypes.c_int64(self.delivered)
        released = ctypes.c_int32(-1)
        free = np.full(self.C, -1, dtype=np.int32)
        rc = self.lib.wrnn_debug_live_batched_deliver(
            self.x.ctypes.data, self.max_steps, progress.ctypes.data, self.C, self.ticket, self.T, self.target,
            self.overlap, self.slots.ctypes.data, self.n_seg, HOP, int(self.mu_law), self.n_classes, ctypes.byref(d),
            ctypes.byref(released), free.ctypes.data, self.wav.ctypes.data)
        assert rc == 0, self.lib.wrnn_last_error()
        assert d.value >= self.delivered
        self.delivered = d.value
        return bool(released.value), free

    def counts(self, counts, retired=()):
        return self.deliver([_word(self.lib, self.ticket, c, b in retired) for b, c in enumerate(counts)])


GEOMETRIES = [
    # T, target, overlap, slots of the folds (non-consecutive, out of order), C
    (30, 2000, 137, [5, 0, 3, 6], 8),        # stride % hop != 0; the last fold runs past T * hop
    (25, 11000, 550, [2], 4),                # one fold, the default geometry
    (40, 2200, 220, [1, 0, 4, 2, 7], 8),     # smoke()'s geometry
    (21, 46, 46, None, 64),                  # 63 folds of 138 samples in a session of 64 slots
]


@pytest.mark.parametrize("mode,mu_law", [("MOL", False), ("RAW", True), ("RAW", False)])
@pytest.mark.parametrize("T,target,overlap,slots,C", GEOMETRIES)
def test_complete_ticket_equals_the_oracle_epilogue(lib, mode, mu_law, T, target, overlap, slots, C):
    n_seg, _ = O.fold_geometry(T * HOP, target, overlap)
    if slots is None:
        slots = list(np.random.RandomState(T).permutation(C)[:n_seg])
    tk = Ticket(lib, T, target, overlap, slots, C, mode, mu_law, seed=T)
    released, free = tk.counts([tk.seg_len] * n_seg, retired=range(n_seg))
    assert released and tk.delivered == tk.wave_len
    assert free.tolist() == [1] * C
    want = tk.want()
    assert np.array_equal(tk.wav.view(np.int64), want.view(np.int64))


@pytest.mark.parametrize("mode,mu_law", [("MOL", False), ("RAW", True)])
def test_partial_counts_deliver_exactly_the_final_prefix(lib, mode, mu_law):
    """Fold 0 ahead, a middle fold lagging, folds in non-consecutive slots: n_ready is exactly the longest prefix whose
    samples every covering fold has published, and every delivered prefix is the final waveform's."""
    tk = Ticket(lib, 40, 2000, 137, [6, 1, 4, 0, 7, 3], 8, mode, mu_law, seed=4)
    want = tk.want()
    rs = np.random.RandomState(5)
    counts = [0] * tk.n_seg
    history = []
    for step in range(400):
        b = rs.randint(tk.n_seg)
        lead = 3 if b == 0 else (1 if b == 2 else 2)              # fold 0 ahead, fold 2 lagging
        counts[b] = min(tk.seg_len, counts[b] + 64 * lead * rs.randint(1, 4))
        admitted = [c > 0 or k == 0 for k, c in enumerate(counts)]  # a fold not yet admitted: its slot's old word
        words = [_word(lib, tk.ticket, c) if a else _word(lib, 3, 64, True) for c, a in zip(counts, admitted)]
        released, _ = tk.deliver(words)
        assert not released
        assert tk.delivered == tk.prefix(counts), (counts, tk.delivered)
        assert np.array_equal(tk.wav[:tk.delivered].view(np.int64), want[:tk.delivered].view(np.int64))
        assert np.isnan(tk.wav[tk.delivered:]).all()                  # nothing past the prefix is written
        history.append(tk.delivered)
        if min(counts) == tk.seg_len:
            break
    assert history == sorted(history) and history[-1] == tk.wave_len
    assert any(0 < h < tk.wave_len for h in history)


def test_delivered_samples_are_never_rewritten(lib):
    tk = Ticket(lib, 30, 2000, 137, [3, 1, 0, 2], 4, seed=6)
    tk.counts([640, 640, 0, 0])
    assert tk.delivered == 640
    tk.wav[:640] = 7.0
    tk.counts([2274, 640, 0, 0])
    assert tk.delivered == tk.stride + 640 and (tk.wav[:640] == 7.0).all()


def test_slots_are_released_together_only_when_every_fold_has_retired(lib):
    tk = Ticket(lib, 30, 2000, 137, [5, 0, 3, 6], 8, seed=7)
    full = [tk.seg_len] * tk.n_seg
    for retired in [(), (0,), (0, 1, 2), (1, 2, 3)]:
        released, free = tk.counts(full, retired=retired)
        assert not released and free.tolist() == [0 if s in (0, 3, 5, 6) else 1 for s in range(8)], retired
    assert tk.delivered == tk.wave_len                            # every sample final, the slots still held
    released, free = tk.counts(full, retired=range(tk.n_seg))
    assert released and free.tolist() == [1] * 8


def test_cancelled_ticket_is_released_with_the_prefix_its_folds_reached(lib):
    """Folds cut short at a boundary retire with the counts they reached: the ticket is released with the longest final
    prefix, which is the reference's."""
    tk = Ticket(lib, 30, 2000, 137, [5, 0, 3, 6], 8, seed=8)
    counts = [1280, 1216, 1216, 1152]
    released, _ = tk.counts(counts, retired=range(tk.n_seg))
    assert released and tk.delivered == tk.prefix(counts) == 1280
    assert np.array_equal(tk.wav[:1280].view(np.int64), tk.want()[:1280].view(np.int64))


def _relaunch(lib, words, slots, posted, cancelled=False, T=30, target=2000, overlap=137, ticket=9):
    """The relaunch decision for one ticket of a session of len(words) slots whose launch has exited."""
    C = len(words)
    progress = np.ascontiguousarray(words, dtype=np.uint64)
    sl = np.ascontiguousarray(slots, dtype=np.int32)
    req, entry = np.zeros(C, np.uint64), np.zeros((C, 4), np.int64)
    launch, released = ctypes.c_int32(-1), ctypes.c_int32(-1)
    rc = lib.wrnn_debug_live_batched_relaunch(progress.ctypes.data, C, ticket, T, target, overlap, sl.ctypes.data, len(slots),
                                              posted, int(cancelled), HOP, req.ctypes.data, entry.ctypes.data,
                                              ctypes.byref(launch), ctypes.byref(released))
    return rc, [int(w) for w in progress], [int(r) for r in req], entry.tolist(), launch.value, released.value


def test_relaunch_admits_the_folds_a_finished_launch_did_not(lib):
    """A launch can exit between two folds' posts (it stops at a boundary where no slot is held).  At the relaunch, folds
    that carry the ticket's tag and the retired bit have finished; folds whose slot carries another tag go into version -1
    of the table at step 0, each with its own fold, rows and the ticket's tag; a fold with the ticket's tag that is not
    retired is an error; a cancelled ticket withdraws its unadmitted folds and is released."""
    tag, stride, seg_len = lib.wrnn_debug_live_tag(9), 2137, 2274
    old = _word(lib, 3, 64, True)                              # an earlier occupant's retired word
    slots = [5, 0, 3, 6]                                       # 4 folds of 30 frames at (2000, 137)
    words = [old] * 8
    words[5] = _word(lib, 9, seg_len, True)                    # fold 0: served by the launch that exited
    words[0] = _word(lib, 9, seg_len, True)                    # fold 1 too
    rc, prog, req, entry, launch, released = _relaunch(lib, words, slots, posted=3)
    assert rc == 0 and launch == 1 and released == 0
    assert entry[3] == [seg_len, 2, 2 * stride, 30 * HOP - 2 * stride]   # fold 2, posted but not admitted
    assert entry[6] == [0, 0, 0, 0] and entry[5] == entry[0] == [0, 0, 0, 0]   # fold 3 not posted; 0, 1 finished
    assert prog[3] == tag << 32 and prog[5] == words[5] and prog[0] == words[0] and prog[6] == old
    rc, *_ = _relaunch(lib, words, slots, posted=4)
    assert rc == 0
    # every posted fold finished, fold 3 not yet posted: no launch until it is
    rc, _, _, entry, launch, released = _relaunch(lib, words, slots, posted=2)
    assert rc == 0 and launch == 0 and released == 0 and all(e == [0, 0, 0, 0] for e in entry)
    # cancelled: the unadmitted folds are withdrawn (their mailbox's tag set back to the slot's word) and the ticket released
    rc, prog, req, entry, launch, released = _relaunch(lib, words, slots, posted=3, cancelled=True)
    assert rc == 0 and launch == 0 and released == 1 and req[3] == 3 and all(e == [0, 0, 0, 0] for e in entry)
    assert prog == words
    # a fold that still carries the ticket's tag without the retired bit: the launch exited with it held
    held = list(words)
    held[0] = _word(lib, 9, 640)
    rc, *_ = _relaunch(lib, held, slots, posted=3)
    assert rc == cabi.WRNN_E_CUDA and b"still held" in lib.wrnn_last_error()


def _slot(lib, state, seed, b, req, cancel, req_seed=0, steps=1000, fold=0, row0=0, rows=1):
    st = np.ascontiguousarray(state, dtype=np.int64)
    sd = ctypes.c_uint64(seed)
    words = np.zeros(2, dtype=np.uint64)
    assert lib.wrnn_debug_live_session_fold_slot(st.ctypes.data, ctypes.byref(sd), b, req, cancel, req_seed, steps, fold,
                                                 row0, rows, words.ctypes.data) == 0, lib.wrnn_last_error()
    return list(st), sd.value, [int(w) for w in words]


def test_slot_decisions_for_a_folded_occupant(lib):
    """A fold is admitted with its fold index and rows, retired SES_DRAIN steps after its end and cancelled at the next
    boundary, as an unbatched occupant is; an occupant's fields stay until the next admission."""
    free = [0, 0, 0, 1, 0, 0, 0]                             # tag, a, e, retired, fold, row0, rows
    s, seed, w = _slot(lib, free, 0, 128, req=5, cancel=0, req_seed=2**40 + 1, steps=2274, fold=3, row0=12 * 3 * HOP + 6411,
                       rows=30 * HOP - 6411)
    assert s == [5, 192, 192 + 2274, 0, 3, 12 * 3 * HOP + 6411, 30 * HOP - 6411] and seed == 2**40 + 1
    assert w == [0, 5 << 32]
    s2, _, w = _slot(lib, s, seed, 192, req=5, cancel=0, fold=7, row0=1, rows=1)   # the occupant's own tag: no new request
    assert s2 == s and w == [0, 0]
    s3, _, w = _slot(lib, s, seed, 2496, req=6, cancel=0, steps=500, fold=1, row0=9, rows=40)   # 2466 + 4 <= 2496
    assert w == [(5 << 32) | RETIRED | 2274, 6 << 32] and s3 == [6, 2560, 3060, 0, 1, 9, 40]
    s4, _, w = _slot(lib, s3, 0, 2624, req=6, cancel=6)      # cancelled mid-fold: ends at the next boundary
    assert s4 == [6, 2560, 2688, 0, 1, 9, 40] and w == [0, 0]
    s5, _, w = _slot(lib, s4, 0, 2752, req=6, cancel=6)
    assert s5[3] == 1 and s5[4:] == [1, 9, 40] and w[0] == (6 << 32) | RETIRED | 128


def test_refusals_without_a_device(lib):
    def refused(rc, match):
        msg = lib.wrnn_last_error().decode()
        assert rc == cabi.WRNN_E_INVALID and match in msg, (rc, msg)
    tk = ctypes.c_int64(-1)
    u = cabi.WrnnUtterance(0x1000, 26, 1, 0x1000)
    sub = lib.wrnn_live_submit_batched
    refused(sub(None, None, 2000, 137, ctypes.byref(tk)), "null utterance or ticket")
    refused(sub(None, ctypes.byref(u), 2000, 137, None), "null utterance or ticket")
    refused(sub(None, ctypes.byref(cabi.WrnnUtterance(None, 26, 1, 0x1000)), 2000, 137, ctypes.byref(tk)), "mel and wav")
    refused(sub(None, ctypes.byref(cabi.WrnnUtterance(0x1000, 20, 1, 0x1000)), 2000, 137, ctypes.byref(tk)), "T must be >= 21")
    for target, overlap in [(0, 137), (2000, 0), (-5, 10), (10, -1)]:
        refused(sub(None, ctypes.byref(u), target, overlap, ctypes.byref(tk)), "target > 0 and overlap > 0")
    refused(sub(None, ctypes.byref(u), 2000, 137, ctypes.byref(tk)), "null handle")
    assert tk.value == -1
    # the delivery hook refuses a fold count other than fold_with_overlap's, a repeated slot and a fold past its row
    x, wav, p = np.zeros((4, 3000), np.float32), np.zeros(29 * HOP), np.zeros(4, np.uint64)
    d, r, f = ctypes.c_int64(0), ctypes.c_int32(0), np.zeros(4, np.int32)
    hook = lib.wrnn_debug_live_batched_deliver

    def call(slots, max_steps=3000):
        sl = np.asarray(slots, np.int32)
        return hook(x.ctypes.data, max_steps, p.ctypes.data, 4, 1, 30, 2000, 137, sl.ctypes.data, len(slots), HOP, 0, 30,
                    ctypes.byref(d), ctypes.byref(r), f.ctypes.data, wav.ctypes.data)
    assert call([0, 1, 2, 3]) == 0
    assert call([0, 1, 2]) == cabi.WRNN_E_INVALID
    assert call([0, 1, 1, 3]) == cabi.WRNN_E_INVALID
    assert call([0, 1, 2, 3], max_steps=2273) == cabi.WRNN_E_INVALID


if __name__ == "__main__":
    sys.exit(pytest.main([__file__, "-v", "-s"]))
