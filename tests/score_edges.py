"""The designed grid of the scoring edge tests: logit vectors (the fc3 bias of a crafted model, so every engine's logits
are these exactly) and the targets scored under each.  Shared by tests/test_score_edges.py (the restatement against the
reference's own loss, tests/golden/score_edge_pins.npz) and tests/test_gpu_score_edges.py (every scoring kernel).

MoL: 14 vectors of 30 logits [10 mixture | 10 means | 10 log-scales].  A "leader" is a component whose mixture logit is
the maximum (+60 against 0 for the others, or tied): every regime has a vector whose leaders take it, so the loss
measures that branch directly.  Components that are not set otherwise copy the first leader's mean and log-scale.
RAW: 6 vectors of 512 logits, each scored on every class's label_2_float(k) and on clamped and half-way targets.

Everything is deterministic (fixed seeds, exact float32 searches); nothing here imports the reference."""
from __future__ import annotations

import numpy as np

F32 = np.float32
HALF_BIN = F32(1.0 / 65535.0)                   # 1. / (num_classes - 1) as torch rounds it
LSM = F32(np.log(1e-14))                         # log_scale_min as a float32 clamp bound
P999 = F32(0.999)
TWENTY = F32(20)
SP20 = (np.nextafter(TWENTY, F32(0)), TWENTY, np.nextafter(TWENTY, F32(40)))   # the softplus threshold and its ulps


def up(x, n=1):
    for _ in range(n):
        x = np.nextafter(F32(x), F32(np.inf))
    return F32(x)


def down(x, n=1):
    for _ in range(n):
        x = np.nextafter(F32(x), F32(-np.inf))
    return F32(x)


# every MoL vector scores these: both edge branches and their float32 thresholds with one ulp to each side
EDGE_Y = [F32(-1), F32(1), P999, -P999, up(P999), down(P999), down(-P999), up(-P999), F32(0.0), F32(-0.0)]


def f32_range(lo, hi):
    """Every float32 in [lo, hi], ascending (lo and hi of one sign)."""
    lo, hi = F32(lo), F32(hi)
    assert lo <= hi and (lo > 0) == (hi > 0)
    if hi <= 0:
        return -f32_range(-hi, -lo)[::-1]
    a, b = np.array([lo, hi], F32).view(np.int32)
    return np.arange(a, b + 1, dtype=np.int32).view(F32)


def args_unit_scale(y, mean):
    """(plus_in, min_in, mid_in) of a component of log-scale 0 (inv_stdv = exp(-0) = 1) in float32, as the kernel and
    the reference evaluate them."""
    c = (y - F32(mean)).astype(F32)
    return (c + HALF_BIN).astype(F32), (c - HALF_BIN).astype(F32), c


def pick_args(ys, arg, want, per=3):
    """Up to `per` targets of ys whose float32 argument equals each value of `want`."""
    out = []
    for w in want:
        hit = ys[arg == w]
        assert hit.size, w
        out += list(hit[np.linspace(0, hit.size - 1, min(per, hit.size)).astype(int)])
    return out


def _vec(mix, means, ls):
    return np.concatenate([np.asarray(mix, F32), np.asarray(means, F32), np.asarray(ls, F32)]).astype(F32)


def _lead(mean, ls, mix=None):
    """Mixture logits `mix`, or 60 on component 0 against 0; every component at (mean, ls)."""
    m = np.zeros(10, F32) if mix is None else np.asarray(mix, F32)
    if mix is None:
        m[0] = 60
    return m, np.full(10, mean, F32), np.full(10, ls, F32)


def exact_half_bin_means():
    """Means m for which y = m +- half_bin are float32 and y - m is exactly +-half_bin (so min_in / plus_in = 0)."""
    ms = [F32(0), HALF_BIN, -HALF_BIN, F32(2.0 ** -17), F32(-2.0 ** -17)]
    for m in ms:
        for s in (1, -1):
            y = F32(m + s * HALF_BIN)
            assert F32(y - m) == s * HALF_BIN, m
    return ms


def sweep_targets(mean, ls):
    """Targets whose cdf_delta (float64) sweeps across 1e-5 on both sides of the mean, and the float32 targets
    closest to each crossing."""
    inv = np.exp(-np.float64(ls))
    ys = []
    for side in (1, -1):
        for x in np.linspace(6.5, 9.5, 25):
            ys.append(F32(mean + side * x / inv))
        # the crossing itself: the float32 targets around where cdf_delta == 1e-5
        a, b = sorted((F32(mean + side * 7.8 / inv), F32(mean + side * 8.4 / inv)))
        cand = f32_range(a, b).astype(np.float64)
        c = cand - np.float64(F32(mean))
        d = 1 / (1 + np.exp(-inv * (c + np.float64(HALF_BIN)))) - 1 / (1 + np.exp(-inv * (c - np.float64(HALF_BIN))))
        k = int(np.argmin(np.abs(d - 1e-5)))
        ys += [F32(v) for v in cand[max(0, k - 6):k + 7]]
    return ys


def mol_grid():
    """[(name, bias (30,), targets (n,))] of the MoL grid."""
    rs = np.random.RandomState(20261017)
    hb_means = exact_half_bin_means()
    V = []

    def add(name, vec, extra):
        ys = EDGE_Y + [F32(v) for v in extra]
        V.append((name, vec.astype(F32), np.array(ys, F32)))

    def mean_targets(m):
        return [m, F32(m + HALF_BIN), F32(m - HALF_BIN)]

    # generic mixture: a dominant component at log-scale -3 among random ones
    mix = np.concatenate([[60], rs.randn(9) * 2]).astype(F32)
    means = np.concatenate([[0], rs.uniform(-1, 1, 9)]).astype(F32)
    ls = np.concatenate([[-3], rs.uniform(-8, 0, 9)]).astype(F32)
    add("generic", _vec(mix, means, ls), mean_targets(F32(0)) + [0.5, -0.5, 0.9, -0.9, 0.3, 0.05])
    # log-scales at the clamp, one ulp to each side, and far below it: means where mean +- half_bin is exact
    for name, l, m in (("clamp", LSM, hb_means[0]), ("clamp+ulp", up(LSM), hb_means[1]), ("clamp-ulp", down(LSM), hb_means[2]),
                       ("ls-40", F32(-40), hb_means[3]), ("ls-100", F32(-100), hb_means[4])):
        add(name, _vec(*_lead(m, l)), mean_targets(m) + [F32(m + 3e-14), F32(m - 7e-14), F32(0.25), F32(-0.6)])
    # wide log-scales and means beyond +-1; the +5 vector's mixture spreads to +-1e4
    mix = np.zeros(10, F32); mix[0], mix[1] = 1e4, -1e4; mix[2:] = rs.randn(8)
    add("ls+5-mean+1.5-spread", _vec(*_lead(1.5, 5.0, mix)), [0.5, -0.5, 0.99, -0.99, 0.1])
    add("ls+20-mean-1.5", _vec(*_lead(-1.5, 20.0)), [0.5, -0.5, 0.99, -0.99, 0.1])
    # cdf_delta across 1e-5 from both sides (log-scale -7)
    m8 = F32(0.2)
    add("cdf-sweep", _vec(*_lead(m8, -7.0)), [m8] + sweep_targets(m8, F32(-7.0)))
    # softplus at 20 +- 1 ulp and above 88.  log_cdf_plus (y < -0.999): component 0 at plus_in ~ 20, component 1 at
    # plus_in ~ 88.5, both leaders; log_pdf_mid: component 2, a third leader at mid_in ~ 20 for y ~ 0.5.
    lo_y = f32_range(F32(-1), down(-P999))
    m_a, m_b, m_c = F32(-20.9995), F32(-89.5), F32(-19.5)
    mid_y = f32_range(F32(0.4999), F32(0.5001))
    y_plus = pick_args(lo_y, args_unit_scale(lo_y, m_a)[0], SP20)
    y_mid = pick_args(mid_y, args_unit_scale(mid_y, m_c)[2], SP20)
    mix, means, ls = _lead(m_a, 0.0)
    mix[1] = mix[2] = 60; means[1], means[2] = m_b, m_c
    add("softplus-cdf_plus-pdf", _vec(mix, means, ls), y_plus + y_mid)
    # log_one_minus_cdf_min (y > 0.999): min_in at 20 +- 1 ulp, then min_in ~ 89.5
    hi_y = f32_range(up(P999), F32(1))
    m_d = F32(-19.0005)
    add("softplus-one_minus-20", _vec(*_lead(m_d, 0.0)), pick_args(hi_y, args_unit_scale(hi_y, m_d)[1], SP20))
    add("softplus-one_minus-88", _vec(*_lead(-88.5, 0.0)), [hi_y[i] for i in (0, 100, 400, 700, 1000)] + [0.5, -0.5])
    # two leaders with means at +-1e4: log_pdf_mid of the first takes softplus(mid_in ~ 1e4)
    mix = np.zeros(10, F32); mix[:2] = 60
    means = np.full(10, -1e4, F32); means[1] = 1e4
    ls = np.zeros(10, F32); ls[1] = 2.0
    add("means+-1e4-split", _vec(mix, means, ls), [0.5, -0.5, 0.9, -0.9, 0.1])
    # a flat mixture (ten exact ties) of random components
    means = rs.uniform(-0.9, 0.9, 10).astype(F32)
    ls = rs.uniform(-6, 0, 10).astype(F32)
    add("flat", _vec(np.zeros(10, F32), means, ls), [means[0], means[3], 0.5, -0.5, 0.7])
    return V


# ---------------------------------------------------------------------------------------------------------------------
# RAW
# ---------------------------------------------------------------------------------------------------------------------
N_CLASSES = 512


def label_2_float(k):
    """utils/dataset.py:88 label_2_float for 9 bits, rounded to float32."""
    return F32(2 * np.asarray(k, np.float64) / (N_CLASSES - 1) - 1)


def raw_label(y):
    """The header's rule: rint((y + 1) * 511 * 0.5) in float32, clamped to [0, 511]."""
    v = np.rint((np.asarray(y, F32) + F32(1)) * F32(N_CLASSES - 1) * F32(0.5))
    return np.clip(v, 0, N_CLASSES - 1).astype(np.int64)


def half_way_targets(ks):
    """For each k, float32 targets y with (y + 1) * 511 * 0.5 == k + 1/2 exactly (the tie rintf breaks to even)."""
    out = []
    for k in ks:
        c = F32(2 * (k + 0.5) / (N_CLASSES - 1) - 1)
        ys = f32_range(down(c, 64), up(c, 64))
        v = (ys + F32(1)).astype(F32) * F32(N_CLASSES - 1)
        v = (v.astype(F32) * F32(0.5)).astype(F32)
        hit = ys[v == F32(k + 0.5)]
        assert hit.size, k
        out.append(hit[hit.size // 2])
    return out


HALF_WAY_K = (256, 100, 333, 400)             # (+0.0 and -0.0 are the half way of 255)


def raw_targets():
    ys = [label_2_float(k) for k in range(N_CLASSES)]
    ys += [F32(-1 - 1 / 511), F32(1 + 1 / 511), F32(1.2), F32(-1.2), F32(1.3), F32(-1.3), F32(0.0), F32(-0.0)]
    ys += half_way_targets(HALF_WAY_K)
    ys = np.array(ys, F32)
    assert np.array_equal(raw_label(ys[:N_CLASSES]), np.arange(N_CLASSES))
    return ys


def raw_grid():
    """[(name, bias (512,), targets (n,))]: every vector is scored on raw_targets()."""
    rs = np.random.RandomState(20261018)
    V = []
    V.append(("normal", rs.randn(512).astype(F32)))
    V.append(("all-equal", np.full(512, 1.5, F32)))
    b = (0.5 * rs.randn(512)).astype(F32); b[[9, 300]] = 5.0          # tied maxima in CTAs 2 and 75
    V.append(("tied-max-2-ctas", b))
    b = (30 * rs.randn(512)).astype(F32); b[77] = 80.0; b[401] = -80.0
    V.append(("x30-spread+-80", b))
    b = rs.randn(512).astype(F32); b[100] = 1e4; b[400] = -1e4
    V.append(("+-1e4", b))
    b = rs.randn(512).astype(F32); b[450] = 30.0                        # maximum in the last quarter of the CTAs
    V.append(("max-in-quarter-3", b))
    ys = raw_targets()
    return [(n, v, ys) for n, v in V]
