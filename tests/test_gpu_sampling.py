"""Every engine form's in-kernel draws and samplers against plain host restatements (oracle/philox.py and
utils/distribution.py:106-121 / fatchord_version.py:231-235 evaluated in float64):

a. MoL Philox draws == the same draws passed in as `uniforms`, bit for bit (keying and word -> uniform map);
b. RAW Philox picks == argmax over the kernel's own logits and the restated Exp(1) draws;
c. the samplers at their edges, on crafted logits (fc3 weight 0, so the logits are fc3's bias exactly);
d. the seed-220 job, whose draw at (fold 0, step 29, class 489) used to be -0.0.

Every job uses seg_first != 0, a seed above 2^32 and philox_offset != 0 unless it restates a fixed job.
Run on a GPU: pytest -m gpu."""
import numpy as np
import pytest
import torch

import helpers
from oracle import contract as C
from oracle import philox as P
from oracle import wavernn_oracle as O
from wavernn_b200 import cabi

pytestmark = pytest.mark.gpu

SEED, OFFSET, SEG_FIRST = (5 << 32) | 7, 0x1234, 77
STRIDE = 20
LOG_SCALE_MIN = np.float32(np.log(1e-14))        # the reference clamps a float32 tensor: its bound is log(1e-14) in float32
# documented accuracy of logf (CUDA C Programming Guide, "Mathematical Functions"): libm logf 1 ulp; the SFU intrinsic
# __logf an absolute 2^-21.41 for x in [0.5, 2] and 3 ulp elsewhere
LIBM, SFU = (None, 1), (2.0 ** -21.41, 3)

# (id, engine, precision, folds, WRNN_STREAM_NF, WRNN_STREAM_CL)
FORMS = {
    "tc-small": ("tcgen05", "fp16", 5, None, None),       # one tile of <= 24 folds
    "tc-big": ("tcgen05", "fp16", 40, None, None),        # one BIG tile (25 .. 64 folds)
    "tc-tiles": ("tcgen05", "fp16", 70, None, None),      # tiles of 64 + 6 folds
    "tc-small-bf16": ("tcgen05", "bf16", 5, None, None),
    "tc-big-bf16": ("tcgen05", "bf16", 40, None, None),
    "tc-tiles-bf16": ("tcgen05", "bf16", 70, None, None),
    "stream-16x1": ("stream", "fp16", 40, "16", "1"),
    "stream-16x4": ("stream", "fp16", 40, "16", "4"),
    "stream-32x1": ("stream", "fp16", 40, "32", "1"),
    "stream-32x4": ("stream", "fp16", 40, "32", "4"),
    "stream-32x4-bf16": ("stream", "bf16", 40, "32", "4"),
    "simt-fp16": ("simt", "fp16", 40, None, None),
    "simt-fp32": ("simt", "fp32", 40, None, None),
    "simt-bf16": ("simt", "bf16", 40, None, None),
}
MOL_FORMS = list(FORMS)
RAW_FORMS = [f for f in FORMS if not f.startswith("stream")]     # the stream engine has no RAW head


def engine_name(form):
    """The name the engine of `form` reports."""
    engine, precision, _, _, cl = FORMS[form]
    return {"tcgen05": f"tcgen05-{precision}", "simt": f"simt-{precision}",
            "stream": f"tcgen05-stream-x4-{precision}" if cl == "4" else f"tcgen05-stream-{precision}"}[engine]


class Runner:
    """One engine on cuda:0, running jobs with every output read back (logits_out pre-filled with NaN)."""

    def __init__(self, model, form, monkeypatch):
        engine, precision, self.n_seg, nf, cl = FORMS[form]
        for var, v in (("WRNN_STREAM_NF", nf), ("WRNN_STREAM_CL", cl)):
            if v is None:
                monkeypatch.delenv(var, raising=False)
            else:
                monkeypatch.setenv(var, v)
        self.form, self.n_classes = form, model.n_classes
        self.eng = cabi.Engine(model.hot_state(), n_classes=model.n_classes, mode=model.mode, precision=precision,
                               engine=engine, device=0)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.eng.close()

    def __call__(self, m_up, aux, steps, *, seg_first=SEG_FIRST, uniforms=None, expo=None, seed=SEED, offset=OFFSET,
                 x_force=None):
        dev = torch.device("cuda", 0)
        t = lambda a: None if a is None else torch.as_tensor(np.ascontiguousarray(a, dtype=np.float32), device=dev)
        p = lambda a: 0 if a is None else a.data_ptr()
        d_m, d_a, d_u, d_e, d_x = t(m_up), t(aux), t(uniforms), t(expo), t(x_force)
        B = self.n_seg
        out = torch.full((B, steps), float("nan"), device=dev)
        lg = torch.full((steps, B, self.n_classes), float("nan"), device=dev)
        self.eng.generate(mels_up=p(d_m), aux=p(d_a), L=m_up.shape[0], n_seg=B, seg_len=steps, seg_stride=STRIDE,
                          out=p(out), seg_first=seg_first, steps=steps, uniforms=p(d_u), expo=p(d_e), philox_seed=seed,
                          philox_offset=offset, x_force=p(d_x), logits_out=p(lg),
                          stream=torch.cuda.current_stream(dev).cuda_stream)
        torch.cuda.synchronize(dev)
        self.eng.check()
        assert self.eng.name == engine_name(self.form), (self.form, self.eng.name)
        res, lgs = out.cpu().numpy(), lg.cpu().numpy()
        assert not np.isnan(res).any() and not np.isnan(lgs).any(), "outputs left unwritten"
        return res, lgs


def inputs(n_seg, steps, seed=0):
    rs = np.random.RandomState(seed)
    L = (n_seg - 1) * STRIDE + steps
    return rs.rand(L, 80).astype(np.float32), rs.randn(L, 128).astype(np.float32)


def crafted(mode, bias):
    """Random-init model whose fc3 is weight 0 and bias `bias`: the logits are `bias` at every fold and step."""
    model = helpers.make_model(0, mode, "cuda")
    with torch.no_grad():
        model.fc3.weight.zero_()
        model.fc3.bias.copy_(torch.as_tensor(bias, dtype=torch.float32))
    return model


@pytest.fixture(scope="module")
def mol_model():
    return helpers.make_model(0, "MOL", "cuda")


@pytest.fixture(scope="module")
def raw_model():
    return helpers.make_model(0, "RAW", "cuda")


def log_err(u, acc):
    """Bound on |computed - exact| of log(u) for a logf with accuracy `acc` = (absolute error on [0.5, 2] or None, ulps)."""
    absolute, ulps = acc
    y = np.abs(np.log(u))
    e = ulps * 2.0 ** -23 * y                   # ulp(y) <= 2^-23 |y|
    if absolute is not None:
        e = np.where((u >= 0.5) & (u <= 2.0), absolute, e)
    return e


def gumbel_err(u, acc):
    """Bound on the error of log(-log u) computed with two such logfs (one rounding of each result included)."""
    lnu = np.abs(np.log(u))
    e1 = log_err(u, acc)
    inner = np.where(e1 < lnu, -np.log1p(-np.minimum(e1 / lnu, 1 - 1e-12)), np.inf)
    v = lnu
    return inner + log_err(v, acc) + 2.0 ** -24 * np.abs(np.log(v))


# ---------------------------------------------------------------------------------------------------------------------
# a. MoL: Philox draws == resident draws
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("form", MOL_FORMS)
def test_mol_philox_draws_equal_the_restated_draws_passed_as_uniforms(form, mol_model, monkeypatch):
    steps = 24
    with Runner(mol_model, form, monkeypatch) as run:
        B = run.n_seg
        m_up, aux = inputs(B, steps)
        out_p, lg_p = run(m_up, aux, steps)
        U = P.mol_uniforms(SEED, OFFSET, SEG_FIRST, B, steps)
        out_u, lg_u = run(m_up, aux, steps, uniforms=U)
        # draws keyed by another seg_first change the samples: the comparison is not vacuous
        out_w, _ = run(m_up, aux, steps, uniforms=P.mol_uniforms(SEED, OFFSET, 0, B, steps))
    same = (out_p == out_u).mean()
    print(f"{form}: Philox run vs restated uniforms: identical samples {same:.4f}, logits {(lg_p == lg_u).mean():.4f}")
    assert np.array_equal(out_p, out_u) and np.array_equal(lg_p, lg_u)
    assert not np.array_equal(out_w, out_p)
    if form in ("tc-small", "stream-16x1"):            # the timed path against the engine contract
        w = O.hot_weights(helpers.state_numpy(mol_model))
        emu, lemu = C.generate_segments(w, m_up, aux, n_seg=B, seg_len=steps, seg_stride=STRIDE, uniforms=U,
                                        precision="fp16", want_logits=True)
        print(f"{form}: vs contract emulation {np.abs(out_p - emu).max():.3e}, logits {np.abs(lg_p - lemu).max():.3e}")
        assert np.abs(out_p - emu).max() <= 1e-3 and np.abs(lg_p - lemu).max() <= 1e-3


# ---------------------------------------------------------------------------------------------------------------------
# b. RAW: Philox picks == host picks from the kernel's logits and the restated draws
# ---------------------------------------------------------------------------------------------------------------------
def raw_host_picks(lg, expo):
    """argmax over classes of log softmax(l) - log e, i.e. of softmax(l) / e (the SIMT engine's form) and of l - log e
    (the persistent engine's form): the same order.  Returns picks (S, B) and the top-two margin."""
    with np.errstate(divide="ignore"):
        sc = lg.astype(np.float64) - np.log(expo.astype(np.float64))
    pick = np.argmax(sc, axis=-1)
    top2 = np.sort(sc, axis=-1)[..., -2:]
    return pick, top2[..., 1] - top2[..., 0]


def kernel_picks(out, n_classes=512):
    k = (out.T.astype(np.float64) + 1.0) * (n_classes - 1) / 2.0
    assert np.abs(k - np.rint(k)).max() <= 1e-3
    return np.rint(k).astype(np.int64)


def forced_inputs(B, steps, seed):
    rs = np.random.RandomState(seed)
    return (2.0 * rs.randint(0, 512, (steps, B)) / 511.0 - 1.0).astype(np.float32)


@pytest.mark.parametrize("form", RAW_FORMS)
def test_raw_philox_picks_equal_host_picks_from_the_restated_draws(form, raw_model, monkeypatch):
    steps = 16
    with Runner(raw_model, form, monkeypatch) as run:
        B = run.n_seg
        m_up, aux = inputs(B, steps, 1)
        out, lg = run(m_up, aux, steps, x_force=forced_inputs(B, steps, 2))
    expo, _ = P.raw_expo(SEED, OFFSET, SEG_FIRST, B, steps)
    want, margin = raw_host_picks(lg, expo)
    got = kernel_picks(out)
    clear = margin > 1e-5
    print(f"{form}: {got.size} RAW picks, {int((~clear).sum())} closer than 1e-5, "
          f"{int((got != want)[clear].sum())} differ where clear, {int((got != want).sum())} in all")
    assert clear.mean() >= 0.99 and np.array_equal(got[clear], want[clear])


# ---------------------------------------------------------------------------------------------------------------------
# c. sampler edges on crafted logits
# ---------------------------------------------------------------------------------------------------------------------
# mixture logits (0, 5, 9 equal: exact ties), then per component (mean, log-scale)
MIX = np.array([0.0, 1e-1, 1e-2, 1e-3, 1e-4, 0.0, -1e-4, -1e-3, -1e-2, 0.0], np.float32)
COMP = [(0.0, LOG_SCALE_MIN - 1.0),      # below the clamp: the sample must use log(1e-14)
        (0.0, LOG_SCALE_MIN),            # at the clamp
        (0.0, LOG_SCALE_MIN + 1.0),      # above it
        (1.5, -5.0),                     # mean beyond +1: the sample is exactly +1
        (-1.5, -5.0),                    # beyond -1: exactly -1
        (0.3, 0.0), (0.1, -2.0), (-0.2, -3.0), (0.05, -4.0), (-0.4, -1.5)]
U_LOG = np.array([0.5, 1e-5, 1 - 1e-5, 0.1, 0.9, 0.02, 0.98, 0.25, 0.75, 0.3], np.float32)
U_HI, U_LO = np.float32(1 - 1e-5), np.float32(1e-5)       # the reference's bounds, as float32


def mol_bias():
    return np.concatenate([MIX, np.array([c[0] for c in COMP], np.float32), np.array([c[1] for c in COMP], np.float32)])


def mol_cells(steps, B, seed=0):
    """Per (step, fold): 10 mixture draws + 1 logistic draw, and the kind of case with its required pick (-1: any)."""
    rs = np.random.RandomState(seed)
    n = steps * B
    u = np.empty((n, 11), np.float32)
    need = np.full(n, -1)
    kind = np.empty(n, object)
    pairs = [(0, 1, 1), (0, 2, 2), (0, 3, 3), (0, 4, 4), (0, 6, 0), (0, 7, 0), (0, 8, 0), (5, 4, 4), (9, 6, 9)]
    for i in range(n):
        lo = rs.uniform(1e-5, 0.05, 10).astype(np.float32)
        lo[rs.rand(10) < 0.3] = U_LO
        c = i % 5
        if c == 0:                                   # one clear winner, chosen by its draw
            k = (i // 5) % 10
            u[i, :10] = lo
            u[i, k] = [U_HI, np.float32(0.9), np.float32(0.99)][(i // 50) % 3]
            kind[i], need[i] = "clear", k
        elif c == 1:                                 # exact ties: equal logits and equal draws -> the lowest index
            u[i, :10] = lo
            tie = [(0, 5, 9), (5, 9), (0, 9)][(i // 5) % 3]
            u[i, list(tie)] = [U_HI, np.float32(0.999), np.float32(0.7)][(i // 15) % 3]
            kind[i], need[i] = "tie", tie[0]
        elif c == 2:                                 # near ties: equal draws close to 1, logits 1e-1 .. 1e-4 apart
            a, b, w = pairs[(i // 5) % len(pairs)]
            u[i, :10] = lo
            u[i, [a, b]] = [U_HI, np.float32(1 - 3e-5), np.float32(1 - 1e-4)][(i // 45) % 3]
            kind[i], need[i] = "near", w
        else:                                        # every draw close to 1: the SFU's worst range, random margins
            u[i, :10] = (1.0 - 10.0 ** rs.uniform(-5, -2, 10)).astype(np.float32)
            u[i, :10] = np.minimum(u[i, :10], U_HI)
            kind[i] = "near-1"
        u[i, 10] = U_LOG[(i // 3) % len(U_LOG)]
    return u.reshape(steps, B, 11), need.reshape(steps, B), kind.reshape(steps, B)


def mol_reference(bias, u):
    """utils/distribution.py:106-121 in float64 on the float32 logits and draws; first maximum wins."""
    l = bias.astype(np.float64)
    u = u.astype(np.float64)
    g = l[:10] - np.log(-np.log(u[..., :10]))
    k = np.argmax(g, axis=-1)
    return g, k


def mol_sample_of(bias, k, ul):
    l = bias.astype(np.float64)
    mean, ls = l[10 + k], np.maximum(l[20 + k], np.float64(LOG_SCALE_MIN))
    ul = ul.astype(np.float64)
    d = np.exp(ls) * (np.log(ul) - np.log1p(-ul))
    return np.clip(mean + d, -1, 1), np.maximum(np.abs(mean), np.abs(d)), np.exp(ls)


@pytest.mark.parametrize("form", MOL_FORMS)
def test_mol_sampler_edges_on_crafted_logits(form, monkeypatch):
    steps = 40
    bias = mol_bias()
    model = crafted("MOL", bias)
    with Runner(model, form, monkeypatch) as run:
        B = run.n_seg
        m_up, aux = inputs(B, steps, 3)
        u, need, kind = mol_cells(steps, B)
        U = np.concatenate([u[..., :10].reshape(steps, 10 * B), u[..., 10]], axis=1)
        out, lg = run(m_up, aux, steps, uniforms=U)
    assert (lg == bias).all(), "fc3 weight 0: the logits must be the bias exactly"
    x = out.T                                        # (S, B)
    g, want = mol_reference(bias, u)
    strict = FORMS[form][0] == "simt"
    acc = LIBM if strict else SFU
    err = gumbel_err(u[..., :10].astype(np.float64), acc) + 2.0 ** -23 * (np.abs(g) + np.abs(bias[:10]))
    assert np.array_equal(want[need >= 0], need[need >= 0])     # the cases are what they claim
    # The kernel reports samples, not picks: a sample is consistent with component k if it is within the sampler's
    # tolerance of k's sample (components 0 and 1 share a sample).  libm: 1e-6 of the larger term.  SFU: 1e-5 of it, or
    # the scale times the documented absolute error of __logf(u) - __logf(1 - u), 2 x 2^-21.41 (at u = 0.5 the SFU
    # engines do not return 0 for it, as libm does, but a value inside that bound).
    tol = 1e-6 if strict else 1e-5
    cand, scale, s = (np.stack(a, -1) for a in zip(*[mol_sample_of(bias, np.full(x.shape, k), u[..., 10]) for k in range(10)]))
    dev = np.abs(cand - x[..., None].astype(np.float64))
    rel = dev / np.maximum(scale, 1e-30)
    cons = rel <= tol
    if not strict:
        cons |= dev <= s * 2.0 ** -20.41
    take = lambda a, k: np.take_along_axis(a, k[..., None], -1)[..., 0]
    flip = ~take(cons, want)
    got = np.where(flip, np.argmin(rel, axis=-1), want)
    fixed = need >= 0
    bad = fixed & flip
    assert not bad.any(), [(kind[i], need[i], got[i], x[i]) for i in zip(*np.nonzero(bad))][:5]
    # a pick may differ from the float64 reference only where the documented logf error explains it
    gap = take(g, want) - take(g, got)
    bound = take(err, want) + take(err, got)
    top2 = np.sort(g, axis=-1)
    margin = top2[..., -1] - top2[..., -2]
    near1 = kind == "near-1"
    print(f"{form}: {x.size} cells; samples of another component than float64's pick: {int(flip.sum())} "
          f"(margins {np.round(gap[flip], 5)[:8]}, bounds {np.round(bound[flip], 5)[:8]}); near-1 cells {int(near1.sum())}, "
          f"{int((near1 & (margin < 0.05)).sum())} with margin < 0.05; largest bound on a Gumbel term {err[near1].max():.3e}")
    assert take(cons, got)[flip].all() and (gap <= bound)[flip].all()
    if strict:
        assert not flip.any()
    ok = ~flip
    half = ok & (u[..., 10] == np.float32(0.5))
    e = take(rel, want)[ok & ~half]
    e_half = (take(dev, want) / take(s, want))[half]
    print(f"{form}: sample error relative to the larger term where the picks agree: max {e.max():.3e}, median {np.median(e):.3e}; "
          f"at u = 0.5, |sample - mean| up to {e_half.max():.3e} x the scale")
    assert (ok & (want == 3)).any() and (x[ok & (want == 3)] == 1.0).all() and (x[ok & (want == 4)] == -1.0).all()
    assert half.any()
    if strict:                                                                               # u = 0.5: the mean, bitwise
        assert np.array_equal(x[half], np.clip(bias[10 + want[half]], -1, 1))
    else:
        assert e_half.max() <= 2.0 ** -20.41
    assert (ok & (want == 0) & (u[..., 10] != np.float32(0.5))).any()                       # the clamp is exercised


RAW_TIED = [3, 4, 131, 300, 511]                 # equal maxima in the classes of five different CTAs
RAW_NEVER = 7                                     # logit -1e4


def raw_bias():
    b = np.random.RandomState(5).uniform(-1, 1, 512).astype(np.float32)
    b[RAW_TIED] = 2.0
    b[RAW_NEVER] = -1e4
    return b


def raw_cells(steps, B, seed=0):
    rs = np.random.RandomState(seed)
    e = rs.exponential(size=(steps, B, 512)).astype(np.float32)
    e = np.maximum(e, np.float32(1e-3))
    need = np.full((steps, B), -1)
    for t in range(steps):
        for b in range(B):
            c = (t * B + b) % 4
            if c == 0:                              # five-way tie across CTAs -> class 3
                e[t, b] = np.maximum(e[t, b], 0.5)
                e[t, b, RAW_TIED] = 0.25
                need[t, b] = 3
            elif c == 1:                            # three-way tie -> class 131
                e[t, b] = np.maximum(e[t, b], 0.5)
                e[t, b, RAW_TIED[2:]] = 0.25
                e[t, b, RAW_TIED[:2]] = 1.0
                need[t, b] = 131
            elif c == 2:                            # an explicit +0.0 draw: p / 0 = +inf, that class is picked
                z = (t * 37 + b * 11) % 512
                if z in RAW_TIED or z == RAW_NEVER:
                    z = 200
                e[t, b, z] = 0.0
                need[t, b] = z
            e[t, b, RAW_NEVER] = np.float32(1e-30)   # the tiniest draw still cannot lift a logit of -1e4
    return e, need


@pytest.mark.parametrize("form", RAW_FORMS)
def test_raw_sampler_ties_zero_draws_and_impossible_classes_on_crafted_logits(form, monkeypatch):
    steps = 16
    bias = raw_bias()
    model = crafted("RAW", bias)
    with Runner(model, form, monkeypatch) as run:
        B = run.n_seg
        m_up, aux = inputs(B, steps, 4)
        expo, need = raw_cells(steps, B)
        out, lg = run(m_up, aux, steps, expo=expo)
    assert (lg == bias).all(), "fc3 weight 0: the logits must be the bias exactly"
    got = kernel_picks(out)
    want, margin = raw_host_picks(lg, expo)
    fixed = need >= 0
    assert np.array_equal(want[fixed], need[fixed])
    clear = ~fixed & (margin > 1e-5)
    print(f"{form}: {int(fixed.sum())} tie / zero-draw cells, {int(clear.sum())} random cells with a clear margin, "
          f"{int((~fixed & ~clear).sum())} closer")
    assert np.array_equal(got[fixed], need[fixed]), [(t, b, need[t, b], got[t, b]) for t, b in zip(*np.nonzero(fixed & (got != need)))][:5]
    assert np.array_equal(got[clear], want[clear]) and (got != RAW_NEVER).all()


# ---------------------------------------------------------------------------------------------------------------------
# d. the zero Exp(1) draw of seed 220 (fold 0, step 29, class 489)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("form", RAW_FORMS)
def test_raw_zero_draw_of_seed_220_picks_as_the_host_does(form, raw_model, monkeypatch):
    """Before the draws were clamped into (0, 1), -logf(1.0f) = -0.0 forced class 489 in the persistent engine
    (log(-0) = -inf) and excluded it in the SIMT engine (p / -0 = -inf).  With the random-init logits the smallest
    draw makes 489 the host's pick; with 489's logit at -100 it cannot win."""
    steps, seed, ev = 32, 220, (29, 0, 489)
    low = raw_bias()
    low[489] = -100.0
    expo, words = P.raw_expo(seed, 0, 0, FORMS[form][2], steps)
    assert words[ev] >> 8 == 0xffffff
    for label, model in (("random-init", raw_model), ("logit -100", crafted("RAW", low))):
        with Runner(model, form, monkeypatch) as run:
            B = run.n_seg
            m_up, aux = inputs(B, steps, 6)
            out, lg = run(m_up, aux, steps, seg_first=0, seed=seed, offset=0, x_force=forced_inputs(B, steps, 7))
        want, margin = raw_host_picks(lg, expo)
        got = kernel_picks(out)
        print(f"{form} {label}: at (fold 0, step 29) host {want[29, 0]} (margin {margin[29, 0]:.3f}), kernel {got[29, 0]}")
        assert margin[29, 0] > 1e-3 and got[29, 0] == want[29, 0]
        clear = margin > 1e-5
        assert np.array_equal(got[clear], want[clear])
        assert (want[29, 0] == 489) == (label == "random-init")
