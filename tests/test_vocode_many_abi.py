"""Host side of wrnn_vocode_many, checked without a device: the ctypes mirrors of wrnn_utterance / wrnn_vocode_batch
against the header, and the job the library lays out for a batch (wrnn_debug_vocode_many_plan) against a restatement
built on wavernn_b200.sharding's fold geometry, refusals included."""
import ctypes
import subprocess
import sys

import numpy as np
import pytest

import helpers
from wavernn_b200 import cabi
from wavernn_b200.sharding import fold_geometry, unbatched_geometry

ROOT = helpers.GOLDEN.parent.parent
HOP = 275
FAKE = 0x1000                      # the hook only tests mel / wav against NULL


@pytest.fixture(scope="module")
def lib():
    if not cabi.is_built():
        import __graft_entry__ as g
        g.build()
    return cabi.load()


def test_struct_layouts_match_header(tmp_path):
    fields = {"wrnn_utterance": (cabi.WrnnUtterance, ("mel", "T", "philox_seed", "wav")),
              "wrnn_vocode_batch": (cabi.WrnnVocodeBatch, ("utts", "n_utts", "batched", "target", "overlap", "mu_law"))}
    lines = ["#include <stddef.h>", "#include <stdio.h>", '#include "wavernn_b200.h"', "int main(void) {"]
    for st, (_, names) in fields.items():
        lines.append(f'  printf("{st} %zu\\n", sizeof({st}));')
        lines += [f'  printf("{st}.{n} %zu\\n", offsetof({st}, {n}));' for n in names]
    lines += ["  return 0;", "}"]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines) + "\n")
    exe = tmp_path / "layout"
    subprocess.run(["cc", "-std=c99", "-I", str(ROOT / "include"), "-o", str(exe), str(src)], check=True)
    got = dict(line.split() for line in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    for st, (cls, names) in fields.items():
        assert int(got[st]) == ctypes.sizeof(cls), st
        for n in names:
            assert int(got[f"{st}.{n}"]) == getattr(cls, n).offset, (st, n)
    assert ctypes.sizeof(cabi.WrnnUtterance) == 32 and ctypes.sizeof(cabi.WrnnVocodeBatch) == 32


def _plan(lib, Ts, seeds, batched, target, overlap, hop=HOP):
    """(rc, message, plan) of the hook for utterances of Ts frames."""
    b, keep = cabi.vocode_batch([(FAKE, T, s, FAKE) for T, s in zip(Ts, seeds)], batched=batched, target=target,
                                overlap=overlap)
    geo = np.zeros(7, dtype=np.int64)
    rc = lib.wrnn_debug_vocode_many_plan(hop, ctypes.byref(b), geo.ctypes.data, None, None)
    if rc != 0:
        return rc, lib.wrnn_last_error().decode(), None
    utt = np.zeros((len(Ts), 3), dtype=np.int64)
    folds = np.zeros((geo[0], 4), dtype=np.int64)
    assert lib.wrnn_debug_vocode_many_plan(hop, ctypes.byref(b), geo.ctypes.data, utt.ctypes.data, folds.ctypes.data) == 0
    del keep
    return 0, "", dict(geo=geo, utt=utt, folds=folds)


def _restated(Ts, seeds, batched, target, overlap, hop=HOP):
    """The batch layout of include/wavernn_b200.h (frames, rows, folds, keys, waveform offsets) from sharding."""
    frame0 = np.concatenate([[0], np.cumsum([T + 4 for T in Ts])])
    wav0 = np.concatenate([[0], np.cumsum([(T - 1) * hop for T in Ts])])
    geos = [fold_geometry(T * hop, target, overlap) if batched else unbatched_geometry(T * hop) for T in Ts]
    seg_len = geos[0].seg_len if batched else max(Ts) * hop
    seg_stride = geos[0].seg_stride if batched else seg_len
    fold0, rows = [0], []
    for i, (T, s, g) in enumerate(zip(Ts, seeds, geos)):
        R = int(frame0[i]) * hop
        for j in range(g.n_seg):
            rows.append((R + (j * g.seg_stride if batched else 0), R + T * hop, np.uint64(s).astype(np.int64), j))
        fold0.append(fold0[-1] + g.n_seg)
    geo = (fold0[-1], seg_len, seg_stride, geos[0].overlap if batched else 0, int(frame0[-1]) * hop, max(Ts), int(wav0[-1]))
    utt = np.stack([frame0[:-1], fold0[:-1], wav0[:-1]], 1)
    return geo, utt, np.array(rows, dtype=np.int64)


CASES = [  # Ts, batched, target, overlap
    ((26, 21, 40), True, 2200, 220),
    ((21,), True, 2200, 220),
    ((800, 33, 121, 57, 21), True, 11000, 550),
    ((110, 37, 64), True, 100, 10),           # hundreds of folds: one utterance's folds straddle tiles of 64
    ((26, 21, 40), False, 2200, 220),
    ((21, 300, 22, 150), False, 11000, 550),
    ((50,), False, 0, 0),
]


@pytest.mark.parametrize("Ts,batched,target,overlap", CASES)
def test_plan_matches_restatement(lib, Ts, batched, target, overlap):
    seeds = [(0x9E3779B97F4A7C15 * (i + 3)) % 2 ** 64 for i in range(len(Ts))]      # high bits set: the whole uint64
    rc, msg, p = _plan(lib, Ts, seeds, batched, target, overlap)
    assert rc == 0, msg
    geo, utt, folds = _restated(Ts, seeds, batched, target, overlap)
    assert tuple(p["geo"]) == geo
    assert np.array_equal(p["utt"], utt)
    assert np.array_equal(p["folds"], folds)
    # every fold reads its own utterance's rows, which map to frames inside its own block of T + 4
    ends = list(utt[1:, 1]) + [geo[0]]
    for i, T in enumerate(Ts):
        f = p["folds"][utt[i, 1]:ends[i]]
        assert (f[:, 0] >= utt[i, 0] * HOP).all() and (f[:, 1] == (utt[i, 0] + T) * HOP).all()


@pytest.mark.parametrize("hop", [1, 3, 256, 600])
def test_plan_matches_restatement_at_other_hops(lib, hop):
    """The batch layout at hops other than 275: frame0 * hop rows per utterance, 4 * hop gap rows between them, folds
    scaled to the hop (a padded last fold per utterance), and one fold per utterance unbatched."""
    Ts = (26, 21, 40, 33)
    seeds = [(0x9E3779B97F4A7C15 * (i + 3)) % 2 ** 64 for i in range(len(Ts))]
    for batched, target, overlap in ((True, 8 * hop, max(2, 4 * hop // 5)), (True, 3 * hop, hop), (False, 0, 0)):
        rc, msg, p = _plan(lib, Ts, seeds, batched, target, overlap, hop)
        assert rc == 0, msg
        geo, utt, folds = _restated(Ts, seeds, batched, target, overlap, hop)
        assert tuple(p["geo"]) == geo and np.array_equal(p["utt"], utt) and np.array_equal(p["folds"], folds), (batched, target)
        ends = list(utt[1:, 1]) + [geo[0]]
        for i, T in enumerate(Ts):
            f = p["folds"][utt[i, 1]:ends[i]]
            assert (f[:, 0] >= utt[i, 0] * hop).all() and (f[:, 1] == (utt[i, 0] + T) * hop).all()
            assert i + 1 == len(Ts) or utt[i + 1, 0] * hop - f[0, 1] == 4 * hop          # the gap rows
        if batched:
            assert geo[0] >= 3 * len(Ts)
            assert any(fold_geometry(T * hop, target, overlap).padded_len != T * hop for T in Ts)


@pytest.mark.parametrize("batched", [True, False])
def test_one_utterance_is_the_single_job(lib, batched):
    """A one-utterance batch is wrnn_vocode's job: its fold_geometry, fold b at row b * seg_stride, key (seed, b)."""
    out = (ctypes.c_int64 * 5)()
    for T in (21, 26, 37, 800):
        rc, msg, p = _plan(lib, [T], [77], batched, 2200, 220)
        assert rc == 0, msg
        assert lib.wrnn_debug_fold_geometry(T * HOP, int(batched), 2200, 220, out) == 0
        n_seg, seg_len, seg_stride, overlap, _ = tuple(out)
        assert tuple(p["geo"][:4]) == (n_seg, seg_len, seg_stride, overlap)
        assert np.array_equal(p["folds"][:, 0], np.arange(n_seg) * seg_stride)
        assert (p["folds"][:, 1] == T * HOP).all()
        assert (p["folds"][:, 2] == 77).all() and np.array_equal(p["folds"][:, 3], np.arange(n_seg))
        assert tuple(p["utt"][0]) == (0, 0, 0) and p["geo"][6] == (T - 1) * HOP


def test_refusals(lib):
    def refused(match, Ts, batched=True, target=2200, overlap=220, null=None, hop=HOP):
        utts = [(0 if null == ("mel", i) else FAKE, T, i, 0 if null == ("wav", i) else FAKE) for i, T in enumerate(Ts)]
        b, keep = cabi.vocode_batch(utts, batched=batched, target=target, overlap=overlap)
        geo = np.zeros(7, dtype=np.int64)
        assert lib.wrnn_debug_vocode_many_plan(hop, ctypes.byref(b), geo.ctypes.data, None, None) == cabi.WRNN_E_INVALID
        assert match in lib.wrnn_last_error().decode(), lib.wrnn_last_error()
        del keep
    refused("1 to 65535 utterances", [])
    refused("utterance 2: T must be >= 21", [26, 30, 20, 40])
    refused("utterance 0: T must be >= 21", [5])
    refused("utterance 1: mel and wav are required", [26, 30], null=("mel", 1))
    refused("utterance 2: mel and wav are required", [26, 30, 22], null=("wav", 2))
    refused("target > 0 and overlap > 0", [26], target=0)
    refused("target > 0 and overlap > 0", [26], overlap=0)
    refused("2^31 samples or longer", [2 ** 30 // HOP, 2 ** 30 // HOP])
    b = cabi.WrnnVocodeBatch(None, 2, 1, 2200, 220, 0)              # null utts array
    geo = np.zeros(7, dtype=np.int64)
    assert lib.wrnn_debug_vocode_many_plan(HOP, ctypes.byref(b), geo.ctypes.data, None, None) == cabi.WRNN_E_INVALID
    # the same batches without the fault are accepted
    assert _plan(lib, [26, 30, 21, 40], [0] * 4, True, 2200, 220)[0] == 0
    assert _plan(lib, [26], [0], False, 0, 0)[0] == 0


def test_vocode_many_refuses_null_handle(lib):
    b, keep = cabi.vocode_batch([(FAKE, 26, 0, FAKE)])
    assert lib.wrnn_vocode_many(None, ctypes.byref(b), None) == cabi.WRNN_E_INVALID
    assert lib.wrnn_vocode_many_host(None, ctypes.byref(b)) == cabi.WRNN_E_INVALID
    del keep


if __name__ == "__main__":
    sys.exit(pytest.main([__file__, "-v", "-s"]))
