"""Scoring, checked without a device: the loss restatement (tests/score_oracle.py) against the reference's own loss
functions (tests/golden/score_pins.npz), the bounds the GPU test holds the SIMT fp32 engine to against the reference,
the ctypes mirror of wrnn_score_utt, and the job wrnn_score_many lays out (wrnn_debug_score_many_plan) with its
refusals."""
import ctypes
import subprocess

import numpy as np
import pytest

import helpers
import score_oracle as SO
from oracle import contract as C
from oracle import wavernn_oracle as O
from wavernn_b200 import cabi
from wavernn_b200.sharding import unbatched_geometry

ROOT = helpers.GOLDEN.parent.parent
HOP = 275
FAKE = 0x1000                      # the hook only tests mel / x / nll against NULL
# SIMT fp32 scoring against score_pins.npz (b) (shipped checkpoint, 4 x 12,100 samples) and (c) (random init), in units
# of score_oracle.mol_sensitivity of the run's own logits: at least 4 x the largest such gap between the fp32
# emulation's logits through score_oracle and the fixture (asserted below; measured 5.5e-3 for (b), 4.6e-7 for (c)).
TRAINED_TOL, RAND_TOL = 2.5e-2, 1e-5


@pytest.fixture(scope="module")
def lib():
    if not cabi.is_built():
        import __graft_entry__ as g
        g.build()
    return cabi.load()


@pytest.fixture(scope="module")
def pins():
    return helpers.load_golden("score_pins.npz")


def test_mol_loss_matches_reference(pins):
    y, lg = pins["mol_y"], pins["mol_logits"]
    got = SO.mol_loss(lg, y)
    tol, ambiguous = SO.mol_loss_tolerance(lg, y)
    d = np.abs(got.astype(np.float64) - pins["mol_nll"])
    print(f"MoL loss vs reference: max {d.max():.3e}, worst / tolerance {(d / tol).max():.3f}, "
          f"{int(ambiguous.sum())} samples with cdf_delta at the 1e-5 branch")
    assert (d <= tol).all()
    # every branch is reached: both edges, the cdf_delta branch and the density fallback
    assert (y < np.float32(-0.999)).any() and (y > np.float32(0.999)).any()
    assert ambiguous.any() and (np.abs(y) < 0.999).sum() > 50


def test_raw_loss_matches_reference(pins):
    got = SO.raw_loss(pins["raw_logits"], pins["raw_y"])
    d = np.abs(got.astype(np.float64) - pins["raw_nll"])
    assert (d <= SO.raw_loss_tolerance(pins["raw_logits"])).all(), d.max()
    labels = SO.raw_label(pins["raw_y"], 512)
    assert {0, 511} <= set(labels.tolist())
    assert np.array_equal(SO.raw_label(2 * np.arange(512) / np.float32(511) - 1, 512), np.arange(512))


def test_reference_bounds_from_the_emulation(pins):
    """The fp32 emulation of the engines' arithmetic (contract.generate_segments) + score_oracle against the reference's
    loss: TRAINED_TOL and RAND_TOL are at least 4 x the gaps."""
    sd0 = {k: v.copy() for k, v in helpers.state_numpy(helpers.make_model(0, "MOL", "cpu")).items()}
    model = helpers.make_model(0, "MOL", "cpu")
    model.load_state_dict(helpers.pretrained_state_dict(), strict=False)
    sd = helpers.state_numpy(model)
    g = helpers.load_golden("trained_tacotron.npz")
    mel = helpers.tacotron_mels()[int(g["sentence"])]
    m_up, aux = O.upsample_network(sd, O.pad_time(mel.T, 2).T, pad=2)
    S = g["raw"].shape[1]
    _, lg = C.generate_segments(O.hot_weights(sd), m_up, aux, n_seg=4, seg_len=S, seg_stride=11550, steps=S, mode="MOL",
                                x_force=g["raw"].T.copy(), uniforms=np.full((S, 44), 0.5, np.float32), want_logits=True,
                                precision="fp32")
    nll = SO.mol_loss(lg.reshape(-1, 30), g["raw"].T.reshape(-1)).reshape(S, 4).T
    rel = lambda a, ref, lg: float((np.abs(a.astype(np.float64) - ref) / SO.mol_sensitivity(lg.reshape(-1, 30))).max())
    gap_b = rel(nll.T.reshape(-1), pins["trained_nll"].T.reshape(-1), lg)
    x, rmel = pins["rand_x"], pins["rand_mel"]
    m_up, aux = O.upsample_network(sd0, O.pad_time(rmel.T, 2).T, pad=2)
    _, lg = C.generate_segments(O.hot_weights(sd0), m_up, aux, n_seg=1, seg_len=x.size, seg_stride=x.size, steps=x.size,
                                mode="MOL", x_force=x[:, None].copy(), uniforms=np.full((x.size, 11), 0.5, np.float32),
                                want_logits=True, precision="fp32")
    gap_c = rel(SO.mol_loss(lg.reshape(-1, 30), x), pins["rand_nll"], lg)
    print(f"fp32 emulation vs reference loss: trained {gap_b:.3e} (bound {TRAINED_TOL}), random init {gap_c:.3e} (bound {RAND_TOL})")
    assert 4 * gap_b <= TRAINED_TOL and 4 * gap_c <= RAND_TOL


def test_struct_layout_matches_header(tmp_path):
    names = ("mel", "T", "x", "n", "nll")
    lines = ["#include <stddef.h>", "#include <stdio.h>", '#include "wavernn_b200.h"', "int main(void) {",
             '  printf("size %zu\\n", sizeof(wrnn_score_utt));']
    lines += [f'  printf("{n} %zu\\n", offsetof(wrnn_score_utt, {n}));' for n in names]
    lines += ["  return 0;", "}"]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines) + "\n")
    exe = tmp_path / "layout"
    subprocess.run(["cc", "-std=c99", "-I", str(ROOT / "include"), "-o", str(exe), str(src)], check=True)
    got = dict(line.split() for line in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    assert int(got["size"]) == ctypes.sizeof(cabi.WrnnScoreUtt) == 40
    for n in names:
        assert int(got[n]) == getattr(cabi.WrnnScoreUtt, n).offset, n


def _plan(lib, Ts, ns, hop=HOP, null=None):
    utts = [(FAKE, T, FAKE, n, FAKE) for T, n in zip(Ts, ns)]
    if null is not None:
        i, field = null
        m, T, x, n, o = utts[i]
        utts[i] = (0 if field == "mel" else m, T, 0 if field == "x" else x, n, 0 if field == "nll" else o)
    arr, count = cabi.utt_array(cabi.WrnnScoreUtt, utts)
    geo = np.zeros(5, dtype=np.int64)
    rc = lib.wrnn_debug_score_many_plan(hop, arr, count, geo.ctypes.data, None)
    if rc != 0:
        return rc, lib.wrnn_last_error().decode(), None
    folds = np.zeros((count, 4), dtype=np.int64)
    assert lib.wrnn_debug_score_many_plan(hop, arr, count, geo.ctypes.data, folds.ctypes.data) == 0
    return 0, "", dict(geo=geo, folds=folds)


@pytest.mark.parametrize("Ts,ns,hop", [((30, 45, 25), (8000, 12000, 6875), 275), ((7,), (1,), 275), ((5, 1, 9), (1100, 200, 2475), 275),
                                       ((12, 3), (2400, 600), 200)])
def test_plan_matches_restatement(lib, Ts, ns, hop):
    rc, msg, pl = _plan(lib, Ts, ns, hop)
    assert rc == 0, msg
    # restatement: each utterance the unbatched geometry of its own stream, laid end to end with the 4 frames of zero
    # padding wrnn_conditioning_frames adds; the job runs the longest n steps
    frame0 = np.concatenate([[0], np.cumsum(np.asarray(Ts) + 4)])
    assert list(pl["geo"]) == [len(Ts), max(ns), frame0[-1] * hop, max(Ts), sum(ns)]
    for i, (T, n) in enumerate(zip(Ts, ns)):
        g = unbatched_geometry(T * hop)
        assert g.n_seg == 1 and n <= g.seg_len
        assert list(pl["folds"][i]) == [frame0[i] * hop, frame0[i] * hop + g.seg_len, frame0[i], sum(ns[:i])]


def test_one_utterance_is_the_job_a_caller_builds(lib):
    """One utterance: one fold of n steps over rows 0 .. T*hop of its own stream, i.e. the wrnn_score job with
    n_seg = 1, seg_len = n, rows read as zeros from T*hop on."""
    T, n = 40, 10000
    rc, msg, pl = _plan(lib, (T,), (n,))
    assert rc == 0, msg
    assert list(pl["geo"][:2]) == [1, n] and list(pl["folds"][0][:2]) == [0, T * HOP]


REFUSALS = [
    (dict(Ts=(), ns=()), "1 to 65535 utterances"),
    (dict(Ts=(3,) * 65536, ns=(10,) * 65536), "1 to 65535 utterances"),
    (dict(Ts=(10, 10), ns=(100, 0)), "utterance 1: n must be in"),
    (dict(Ts=(10, 10, 10), ns=(100, 100, 10 * HOP + 1)), "utterance 2: n must be in"),
    (dict(Ts=(10, 10), ns=(100, 100), null=(0, "mel")), "utterance 0: mel, x and nll are required"),
    (dict(Ts=(10, 10), ns=(100, 100), null=(1, "x")), "utterance 1: mel, x and nll are required"),
    (dict(Ts=(10, 10), ns=(100, 100), null=(1, "nll")), "utterance 1: mel, x and nll are required"),
    (dict(Ts=(4_000_000, 4_000_000), ns=(10, 10)), "2^31"),
]


@pytest.mark.parametrize("kw,msg", REFUSALS, ids=[m.split(":")[0] + f"-{i}" for i, (_, m) in enumerate(REFUSALS)])
def test_refusals(lib, kw, msg):
    rc, got, _ = _plan(lib, **kw)
    assert rc == cabi.WRNN_E_INVALID and msg in got, got


def test_null_utterance_array_is_refused(lib):
    geo = np.zeros(5, dtype=np.int64)
    assert lib.wrnn_debug_score_many_plan(HOP, None, 1, geo.ctypes.data, None) == cabi.WRNN_E_INVALID
    assert "non-null utts" in lib.wrnn_last_error().decode()
