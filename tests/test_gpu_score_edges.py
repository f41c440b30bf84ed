"""wrnn_score at the edges of the loss, on every scoring kernel: the grid of tests/score_edges.py, each vector the fc3
bias of a crafted model (fc3 weight 0, so every engine's logits are the bias exactly), against the reference's own loss
pinned in tests/golden/score_edge_pins.npz (tests/test_score_edges.py checks the pins and the grid's coverage on the CPU).

Forms (tests/test_gpu_sampling.py FORMS): persistent fp16 | bf16 at 5, 40 and 70 folds (small tile, BIG tile, 64 + 6
folds over two launches); stream MoL 16 | 32 folds per CTA x 1 | 4 CTAs at fp16 and 32 x 4 at bf16; SIMT fp32 | fp16 |
bf16 at 40 folds (two tiles).  Targets are laid out as x_force[t, b] = grid[(t B + b) mod G] with G coprime with every
fold count, over enough steps that each target lands in several folds, steps and tiles.  Asserted:
  1. logits_out == bias;
  2. nll against the reference pin, and against tests/score_oracle.py on the run's own logits, within
     mol_loss_tolerance / raw_loss_tolerance;
  3. bit-invariance: every cell of one (vector, target) holds the same bits, across folds, steps, tiles and launches;
     MoL across all engines and precisions too (every engine inlines the same mol_nll on the same fp32 logits); RAW
     across the persistent forms (one fixed reduction tree whatever the tile), the SIMT engine, which sums in another
     order, held to the tolerance only.
Each form's worst error / tolerance is printed.
Run on a GPU: pytest -m gpu -s tests/test_gpu_score_edges.py"""
import math

import numpy as np
import pytest
import torch

import score_edges as E
import score_oracle as SO
import helpers
from test_gpu_sampling import FORMS, SEG_FIRST, STRIDE, Runner, crafted, engine_name, inputs

pytestmark = pytest.mark.gpu

MOL_FORMS = ["tc-small", "tc-big", "tc-tiles", "tc-small-bf16", "tc-big-bf16", "tc-tiles-bf16", "stream-16x1",
             "stream-16x4", "stream-32x1", "stream-32x4", "stream-32x4-bf16", "simt-fp32", "simt-fp16", "simt-bf16"]
RAW_FORMS = [f for f in MOL_FORMS if not f.startswith("stream")]
PERSISTENT = [f for f in MOL_FORMS if f.startswith("tc-")]
REPS, MIN_STEPS = 4, 16                    # cells per target and form (at least); steps per job (at least)
WORST = {}                                 # (head, form) -> [worst / tolerance vs the pin, vs the restatement]
MOL_NAMES, RAW_NAMES = [n for n, _, _ in E.mol_grid()], [n for n, _, _ in E.raw_grid()]


class Scorer(Runner):
    """Runner's engine, scoring: nll (S, B) and logits (S, B, classes) of x_force (S, B), both pre-filled with NaN."""

    def score(self, x_force):
        dev = torch.device("cuda", 0)
        S, B = x_force.shape
        m_up, aux = inputs(B, S, 11)
        d_m, d_a, d_x = (torch.as_tensor(a, device=dev) for a in (m_up, aux, np.ascontiguousarray(x_force)))
        nll = torch.full((S, B), float("nan"), device=dev)
        lg = torch.full((S, B, self.n_classes), float("nan"), device=dev)
        self.eng.score(mels_up=d_m.data_ptr(), aux=d_a.data_ptr(), L=m_up.shape[0], n_seg=B, seg_len=S, seg_stride=STRIDE,
                       seg_first=SEG_FIRST, steps=S, x_force=d_x.data_ptr(), nll=nll.data_ptr(), logits_out=lg.data_ptr(),
                       stream=torch.cuda.current_stream(dev).cuda_stream)
        torch.cuda.synchronize(dev)
        self.eng.check()
        assert self.eng.name == engine_name(self.form), (self.form, self.eng.name)
        return nll.cpu().numpy(), lg.cpu().numpy()


def layout(G, B):
    """(grid index per cell (S, B), S): cell (t, b) scores target (t B + b) mod G' of the grid padded to G' >= G entries,
    G' coprime with B, so that a target's cells fall in different folds."""
    Gp = G
    while math.gcd(Gp, B) != 1:
        Gp += 1
    S = max(MIN_STEPS, -(-REPS * Gp // B))
    return (np.arange(S * B).reshape(S, B) % Gp) % G, S


@pytest.fixture(scope="module")
def pins():
    return helpers.load_golden("score_edge_pins.npz")


def run_vector(head, i, pins, forms, monkeypatch):
    """Scores vector i of `head` on every form.  Returns ({form: per-target nll (G,)}, [failures]); every form runs and
    reports before the test asserts, so one run shows every form's state."""
    key = head.lower()
    bias, y, ref = pins[f"{key}_bias_{i}"], pins[f"{key}_y_{i}"], pins[f"{key}_nll_{i}"].astype(np.float64)
    name = str(pins[f"{key}_names"][i])
    G, nc = y.size, bias.size
    model = crafted(head, bias)
    per_target, bad = {}, []
    for form in forms:
        with Scorer(model, form, monkeypatch) as sc:
            idx, S = layout(G, sc.n_seg)
            nll, lg = sc.score(y[idx])
        what = f"{head} '{name}' [{form}]"
        if not (lg == bias).all():
            bad.append((what, "fc3 weight 0: the logits must be the bias exactly"))
            continue
        g, v, ycell, lgc = idx.reshape(-1), nll.reshape(-1), y[idx].reshape(-1), lg.reshape(-1, nc)
        if head == "MOL":
            tol, _ = SO.mol_loss_tolerance(lgc, ycell)
            own = SO.mol_loss(lgc, ycell)
        else:
            tol = SO.raw_loss_tolerance(lgc)
            own = SO.raw_loss(lgc, ycell)
        with np.errstate(invalid="ignore"):
            d_ref = np.where(np.isfinite(v), np.abs(v.astype(np.float64) - ref[g]) / tol, np.inf)
            d_own = np.where(np.isfinite(v), np.abs(v.astype(np.float64) - own) / tol, np.inf)
        w = WORST.setdefault((head, form), [0.0, 0.0])
        w[0], w[1] = max(w[0], d_ref.max()), max(w[1], d_own.max())
        print(f"{what}: {v.size} cells, {S} steps; worst / tolerance vs reference {d_ref.max():.3e}, vs restatement {d_own.max():.3e}")
        if d_ref.max() > 1 or d_own.max() > 1:
            j = np.nonzero((d_ref > 1) | (d_own > 1))[0]
            bad.append((what, "outside the tolerance", [(float(ycell[k]), float(v[k]), float(ref[g[k]]), float(own[k]), float(tol[k]))
                                                        for k in j[:4]]))
        u, pos = np.unique(g, return_index=True)
        assert u.size == G, what
        first = v[pos]                                 # each target's first cell
        same = first[g].view(np.uint32) == v.view(np.uint32)
        if not same.all():
            bad.append((what, "cells of one target differ", [(float(ycell[j]), float(v[j]), float(first[g[j]]))
                                                             for j in np.nonzero(~same)[0][:4]]))
        per_target[form] = first
    return per_target, bad


def same_bits(per_target, forms, what):
    forms = [f for f in forms if f in per_target]
    base = per_target[forms[0]].view(np.uint32)
    bad = []
    for f in forms[1:]:
        diff = per_target[f].view(np.uint32) != base
        if diff.any():
            bad.append((what, f, "differs from", forms[0], "at targets", np.nonzero(diff)[0][:6].tolist(),
                        per_target[f][diff][:3].tolist(), per_target[forms[0]][diff][:3].tolist()))
    return bad


@pytest.mark.parametrize("i", range(len(MOL_NAMES)), ids=MOL_NAMES)
def test_mol_edges_on_every_engine(pins, i, monkeypatch):
    per_target, bad = run_vector("MOL", i, pins, MOL_FORMS, monkeypatch)
    bad += same_bits(per_target, MOL_FORMS, f"MoL '{pins['mol_names'][i]}' across engines")
    assert not bad, bad


@pytest.mark.parametrize("i", range(len(RAW_NAMES)), ids=RAW_NAMES)
def test_raw_edges_on_every_engine(pins, i, monkeypatch):
    per_target, bad = run_vector("RAW", i, pins, RAW_FORMS, monkeypatch)
    bad += same_bits(per_target, PERSISTENT, f"RAW '{pins['raw_names'][i]}' across the persistent forms")
    assert not bad, bad


def test_report_worst_error_per_form():
    """Each form's worst |nll - reference pin| and |nll - restatement on its logits|, in units of the tolerance."""
    if not WORST:
        pytest.skip("run with the vector tests")
    for (head, form), (r, o) in sorted(WORST.items()):
        print(f"score edges {head} {form:18s} ({FORMS[form][1]}): worst / tolerance vs reference {r:.3e}, vs restatement {o:.3e}")
