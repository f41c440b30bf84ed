"""The scoring edge grid on the CPU (tests/score_edges.py against tests/golden/score_edge_pins.npz, the reference's own
discretized_mix_logistic_loss(reduce=False) and F.cross_entropy):

  1. the restatement tests/score_oracle.py matches every pin within half of its tolerance, leaving the other half to the
     device (tests/test_gpu_score_edges.py holds every scoring kernel to the whole tolerance);
  2. coverage: every regime of the loss the grid is built for holds at least 8 cells, classified in float64 by the
     mixture's leading components with the reference's float32 constants, and every cell on the ambiguous 1e-5 band of
     cdf_delta is flagged by mol_loss_tolerance;
  3. negative controls: a restatement that is subtly wrong in one way (a float64 threshold, no clamp, an unthresholded
     softplus, ...) misses the pins by more than the device's tolerance in at least one cell, so the grid would catch a
     kernel wrong in that way."""
import numpy as np
import pytest

import helpers
import score_edges as E
import score_oracle as SO

F32 = np.float32


@pytest.fixture(scope="module")
def pins():
    return helpers.load_golden("score_edge_pins.npz")


def mol_cells(pins):
    """(logits (N, 30), y (N,), reference nll (N,), vector index (N,)) of every MoL cell."""
    L, Y, R, V = [], [], [], []
    for i in range(len(pins["mol_names"])):
        y = pins[f"mol_y_{i}"]
        L.append(np.repeat(pins[f"mol_bias_{i}"][None], y.size, 0)); Y.append(y); R.append(pins[f"mol_nll_{i}"])
        V.append(np.full(y.size, i))
    return np.concatenate(L), np.concatenate(Y), np.concatenate(R).astype(np.float64), np.concatenate(V)


def raw_cells(pins):
    L, Y, R = [], [], []
    for j in range(len(pins["raw_names"])):
        y = pins[f"raw_y_{j}"]
        L.append(np.repeat(pins[f"raw_bias_{j}"][None], y.size, 0)); Y.append(y); R.append(pins[f"raw_nll_{j}"])
    return np.concatenate(L), np.concatenate(Y), np.concatenate(R).astype(np.float64)


def test_pins_are_the_grid(pins):
    """The committed pins were made from this grid: same vectors, same targets, bit for bit."""
    for key, grid in (("mol", E.mol_grid()), ("raw", E.raw_grid())):
        assert list(pins[f"{key}_names"]) == [n for n, _, _ in grid]
        for i, (_, bias, y) in enumerate(grid):
            assert np.array_equal(pins[f"{key}_bias_{i}"].view(np.uint32), bias.view(np.uint32)), (key, i)
            assert np.array_equal(pins[f"{key}_y_{i}"].view(np.uint32), y.view(np.uint32)), (key, i)
    assert all(np.isfinite(pins[k]).all() for k in pins.files if "_nll_" in k)


# ---------------------------------------------------------------------------------------------------------------------
# 1. the restatement against the reference
# ---------------------------------------------------------------------------------------------------------------------
def test_mol_restatement_within_half_the_tolerance(pins):
    lg, y, ref, _ = mol_cells(pins)
    tol, _ = SO.mol_loss_tolerance(lg, y)
    d = np.abs(SO.mol_loss(lg, y).astype(np.float64) - ref)
    print(f"MoL edge grid, {y.size} cells: restatement vs reference worst / tolerance {(d / tol).max():.3e}")
    assert (d <= 0.5 * tol).all(), np.argmax(d / tol)


def test_raw_restatement_within_half_the_tolerance(pins):
    lg, y, ref = raw_cells(pins)
    tol = SO.raw_loss_tolerance(lg)
    d = np.abs(SO.raw_loss(lg, y).astype(np.float64) - ref)
    print(f"RAW edge grid, {y.size} cells: restatement vs reference worst / tolerance {(d / tol).max():.3e}")
    assert (d <= 0.5 * tol).all(), np.argmax(d / tol)


# ---------------------------------------------------------------------------------------------------------------------
# 2. coverage
# ---------------------------------------------------------------------------------------------------------------------
def branch_quantities(lg, y):
    """Per (cell, component), float64 on the float32 logits with the reference's float32 constants: log-scale (clamped),
    mean, plus_in, min_in, mid_in, cdf_plus, cdf_min, and the float32 arguments of the three softplus calls."""
    lg64 = lg.astype(np.float64)
    y64 = y.astype(np.float64)[:, None]
    ls = np.maximum(lg64[:, 20:], np.float64(E.LSM))
    mean = lg64[:, 10:20]
    inv = np.exp(-ls)
    hb = np.float64(E.HALF_BIN)
    q = dict(raw_ls=lg[:, 20:], mean=lg[:, 10:20], plus_in=inv * (y64 - mean + hb), min_in=inv * (y64 - mean - hb),
             mid_in=inv * (y64 - mean))
    with np.errstate(over="ignore"):
        q["cp"], q["cm"] = 1 / (1 + np.exp(-q["plus_in"])), 1 / (1 + np.exp(-q["min_in"]))
        inv32 = np.exp(-np.maximum(lg[:, 20:], E.LSM), dtype=F32)
        c32 = (y[:, None] - lg[:, 10:20]).astype(F32)
        q["plus32"], q["min32"], q["mid32"] = inv32 * (c32 + E.HALF_BIN), inv32 * (c32 - E.HALF_BIN), inv32 * c32
    return q


def regimes(lg, y):
    """name -> mask of cells (N,) whose leading mixture components (logit within 1 of the maximum) take the regime."""
    q = branch_quantities(lg, y)
    mix = lg[:, :10].astype(np.float64)
    lead = mix >= mix.max(1, keepdims=True) - 1
    Y = y[:, None]
    lo, hi = Y < -E.P999, Y > E.P999
    mid = ~lo & ~hi
    d = q["cp"] - q["cm"]
    pdf = mid & (d <= 1e-5)
    sp20 = lambda a: np.isin(a, np.array(E.SP20, F32))
    any_lead = lambda m: (np.broadcast_to(m, lead.shape) & lead).any(1)
    return {
        "y = +-1": np.abs(y) == 1,
        "y = +-float32(0.999)": np.abs(y) == E.P999,
        "y one ulp above float32(0.999)": np.abs(y) == E.up(E.P999),
        "y one ulp below float32(0.999)": np.abs(y) == E.down(E.P999),
        "y = +-0": y == 0,
        "y = mean (mid_in = 0)": any_lead(mid & (Y == q["mean"])),
        "y = mean +- half_bin (min_in or plus_in = 0)": any_lead(mid & ((q["min32"] == 0) | (q["plus32"] == 0))),
        "cdf_delta just above 1e-5": any_lead(mid & (d > 1e-5) & (d <= 3e-5)),
        "cdf_delta just below 1e-5": any_lead(mid & (d <= 1e-5) & (d >= 3e-6)),
        "log-scale = float32(log 1e-14)": any_lead(q["raw_ls"] == E.LSM),
        "log-scale one ulp above the clamp": any_lead(q["raw_ls"] == E.up(E.LSM)),
        "log-scale one ulp below the clamp": any_lead(q["raw_ls"] == E.down(E.LSM)),
        "log-scale -40": any_lead(q["raw_ls"] == -40),
        "log-scale -100": any_lead(q["raw_ls"] == -100),
        "log-scale +5": any_lead(q["raw_ls"] == 5),
        "log-scale +20": any_lead(q["raw_ls"] == 20),
        "softplus(plus_in) at 20 +- 1 ulp (y < -0.999)": any_lead(lo & sp20(q["plus32"])),
        "softplus(min_in) at 20 +- 1 ulp (y > 0.999)": any_lead(hi & sp20(q["min32"])),
        "softplus(mid_in) at 20 +- 1 ulp (log_pdf_mid)": any_lead(pdf & sp20(q["mid32"])),
        "softplus(plus_in) above 88 (y < -0.999)": any_lead(lo & (q["plus_in"] > 88)),
        "softplus(min_in) above 88 (y > 0.999)": any_lead(hi & (q["min_in"] > 88)),
        "softplus(mid_in) above 88 (log_pdf_mid)": any_lead(pdf & (q["mid_in"] > 88)),
        "mean +-1.5": any_lead(np.abs(q["mean"]) == 1.5),
        "mean +-1e4": any_lead(np.abs(q["mean"]) == 1e4),
        "flat mixture (ten exact ties)": (mix == mix[:, :1]).all(1),
        "mixture split evenly between two": lead.sum(1) == 2,
        "mixture spread to +-1e4": (mix.max(1) >= 1e4) & (mix.min(1) <= -1e4),
    }


def test_every_regime_has_cells(pins):
    lg, y, _, _ = mol_cells(pins)
    counts = {k: int(m.sum()) for k, m in regimes(lg, y).items()}
    for k, n in counts.items():
        print(f"{n:4d}  {k}")
    assert all(n >= 8 for n in counts.values()), {k: n for k, n in counts.items() if n < 8}


def test_cells_on_the_1e5_band_are_flagged(pins):
    """A component whose cdf_delta lies within a few float32 ulps of the cdfs from 1e-5 may take either branch in two
    fp32 evaluations: mol_loss_tolerance must flag every such cell (and admit the jump between the branch values)."""
    lg, y, _, _ = mol_cells(pins)
    q = branch_quantities(lg, y)
    d = q["cp"] - q["cm"]
    band = ((np.abs(d - 1e-5) <= 4 * 2.0 ** -24 * np.maximum(q["cp"], q["cm"])) & (np.abs(y[:, None]) <= E.P999)).any(1)
    _, near = SO.mol_loss_tolerance(lg, y)
    print(f"{int(band.sum())} cells on the band, {int(near.sum())} flagged")
    assert band.sum() >= 8 and near[band].all()


def test_raw_grid_coverage(pins):
    """Every class is a target of every vector, so the target's CTA and quarter (CTAs 0-31, 32-63, ...) differ from the
    maximum's in most cells; clamped and half-way targets, ties and +-1e4 logits are present."""
    lg, y, _ = raw_cells(pins)
    lab = SO.raw_label(y, 512)
    assert np.array_equal(lab, E.raw_label(y))
    for j in range(len(pins["raw_names"])):
        assert set(E.raw_label(pins[f"raw_y_{j}"])) == set(range(512))
    top = np.argmax(lg, 1)
    other_q = (top // 128) != (lab // 128)
    tied = (lg == lg.max(1, keepdims=True)).sum(1) >= 2
    v = ((y + F32(1)) * F32(511) * F32(0.5)).astype(np.float64)                    # the label's argument, in float32
    print(f"{y.size} RAW cells: {int(other_q.sum())} with maximum and target in different quarters, {int(tied.sum())} tied")
    assert other_q.sum() >= 8 and tied.sum() >= 8
    assert ((v < -0.5) | (v > 511.5)).sum() >= 8                                    # clamped labels
    k, half = np.floor(v), v == np.floor(v) + 0.5                                  # k + 1/2: rint breaks to even
    assert (half & (k % 2 == 1) & (lab == k + 1)).sum() >= 8 and (half & (k % 2 == 0) & (lab == k)).sum() >= 8
    assert (np.abs(lg).max(1) >= 1e4).sum() >= 8


# ---------------------------------------------------------------------------------------------------------------------
# 3. negative controls
# ---------------------------------------------------------------------------------------------------------------------
def mol_variant(logits, y, *, thr64=False, clamp=True, threshold=True, pdf_offset=True, log_softmax=True):
    """score_oracle.mol_loss with one deliberate defect switched on."""
    lg = np.asarray(logits, dtype=F32)
    y = np.asarray(y, dtype=F32)[:, None]
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        def softplus(x):
            sp = np.log1p(np.exp(x, dtype=F32), dtype=F32)
            return np.where(x > F32(20), x, sp).astype(F32) if threshold else sp
        ls = np.maximum(lg[:, 20:], E.LSM) if clamp else lg[:, 20:]
        c = y - lg[:, 10:20]
        inv = np.exp(-ls, dtype=F32)
        plus_in, min_in, mid_in = inv * (c + E.HALF_BIN), inv * (c - E.HALF_BIN), inv * c
        cdf_delta = F32(1) / (F32(1) + np.exp(-plus_in, dtype=F32)) - F32(1) / (F32(1) + np.exp(-min_in, dtype=F32))
        pdf = mid_in - ls - F32(2) * softplus(mid_in)
        if pdf_offset:
            pdf = pdf - F32(np.log(32767.5))
        inner = np.where(cdf_delta > F32(1e-5), np.log(np.maximum(cdf_delta, F32(1e-12)), dtype=F32), pdf)
        yt = y.astype(np.float64) if thr64 else y
        lp = np.where(yt < -0.999 if thr64 else yt < F32(-0.999), plus_in - softplus(plus_in),
                      np.where(yt > 0.999 if thr64 else yt > F32(0.999), -softplus(min_in), inner))
        if log_softmax:
            pi = lg[:, :10]
            mx = pi.max(1, keepdims=True)
            lp = lp + ((pi - mx) - np.log(np.exp(pi - mx, dtype=F32).sum(1, keepdims=True, dtype=F32), dtype=F32))
        m = lp.max(1)
        return (-(m + np.log(np.exp(lp - m[:, None], dtype=F32).sum(1, dtype=F32), dtype=F32))).astype(F32)


def raw_variant(logits, y, label):
    lg = np.asarray(logits, dtype=F32)
    v = (np.asarray(y, F32) + F32(1)) * F32(511) * F32(0.5)
    k = {"floor": lambda: np.clip(np.floor(v), 0, 511),
         "half away from zero": lambda: np.clip(np.sign(v) * np.floor(np.abs(v) + F32(0.5)), 0, 511),
         "unclamped, wrapped": lambda: np.mod(np.rint(v), 512)}[label]().astype(np.int64)
    mx = lg.max(1)
    s = np.exp(lg - mx[:, None], dtype=F32).sum(1, dtype=F32)
    return (-((lg[np.arange(len(lg)), k] - mx) - np.log(s, dtype=F32))).astype(F32)


MOL_DEFECTS = {"0.999 thresholds compared in float64": dict(thr64=True), "no log-scale clamp": dict(clamp=False),
               "softplus without its threshold": dict(threshold=False),
               "log_pdf_mid without - log(32767.5)": dict(pdf_offset=False),
               "mixture log-softmax left out": dict(log_softmax=False)}


def test_mol_variant_with_no_defect_is_the_restatement(pins):
    lg, y, _, _ = mol_cells(pins)
    assert np.array_equal(mol_variant(lg, y), SO.mol_loss(lg, y))


@pytest.mark.parametrize("defect", list(MOL_DEFECTS))
def test_mol_defect_misses_the_pins(pins, defect):
    lg, y, ref, v = mol_cells(pins)
    tol, _ = SO.mol_loss_tolerance(lg, y)
    with np.errstate(invalid="ignore"):
        got = mol_variant(lg, y, **MOL_DEFECTS[defect]).astype(np.float64)
        miss = ~(np.abs(got - ref) <= tol)                                 # NaN and inf miss
    names = sorted({str(pins["mol_names"][i]) for i in v[miss]})
    print(f"MoL defect '{defect}': {int(miss.sum())} of {y.size} cells miss the pins by more than the tolerance ({names})")
    assert miss.any()


@pytest.mark.parametrize("label", ["floor", "half away from zero", "unclamped, wrapped"])
def test_raw_label_defect_misses_the_pins(pins, label):
    lg, y, ref = raw_cells(pins)
    tol = SO.raw_loss_tolerance(lg)
    miss = np.abs(raw_variant(lg, y, label).astype(np.float64) - ref) > tol
    print(f"RAW label by '{label}': {int(miss.sum())} of {y.size} cells miss the pins by more than the tolerance")
    assert miss.any()
