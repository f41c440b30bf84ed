"""wrnn_epilogue (mu-law expansion, equal-power cross-fade + overlap-add, final fade-out; float64 on the device) at
every geometry its branches distinguish, called directly on synthetic fp32 sample blocks with the tables of
WaveRNN._epilogue_tables, against

  (a) WaveRNN._epilogue, the host numpy restatement, on the same samples: bit for bit;
  (b) wavernn_oracle.epilogue (the reference's xfade_and_unfold + decode_mu_law + fade-out in float64): bit for bit,
      except where the mu-law table differs from the oracle's own expansion (numpy's vectorised np.power may miss the C
      library's pow by 1 ulp, DESIGN §5): those entries within 1 ulp of the power, counted.

The cases cover one, two and 40 folds on the batched path; overlap 1, 2, 3, 275 and 276 (silence overlap // 2); target
1, below the overlap and far above it; the full unfolded length (the last overlap samples clamp to the last fold) and
cropped waves; a fade-out as long as the wave; the unbatched path (no fade tables); a wave over three passes of the
capped grid-stride loop (8 blocks of 256 threads per SM); MoL samples with exact +-1 and +-0; RAW samples holding every
one of the 512 class values 2k / 511 - 1, as the kernels write them, with and without mu-law.  Every refusal of
wrnn_epilogue is run once, each followed by a valid call that must still be exact.  Run on a GPU: pytest -m gpu -s."""
import re
import types

import numpy as np
import pytest
import torch

import kernel_jobs as K
from oracle import wavernn_oracle as O
from wavernn_b200 import cabi

pytestmark = pytest.mark.gpu

N = 512
F32 = np.float32
_models = {}


def model(hop):
    """A small RAW WaveRNN at `hop` (n_classes 512): its _epilogue_tables and _epilogue, with a fade-out of 20 hops."""
    if hop not in _models:
        _models[hop] = K.geometry_model(hop, mode="RAW", rnn_dims=32, fc_dims=32)
        assert _models[hop].n_classes == N and _models[hop].hop_length == hop
    return _models[hop]


def labels_to_samples(k):
    """The fp32 sample the RAW samplers write for class k: 2.0f * (float)k / ((float)n - 1.0f) - 1.0f."""
    return F32(2) * np.asarray(k).astype(F32) / (F32(N) - F32(1)) - F32(1)


def geometry(batched, n_seg, target, overlap, seg_len=None):
    if batched:
        return types.SimpleNamespace(n_seg=n_seg, target=target, overlap=overlap, seg_len=target + 2 * overlap,
                                     seg_stride=target + overlap)
    return types.SimpleNamespace(n_seg=1, target=seg_len, overlap=0, seg_len=seg_len, seg_stride=seg_len)


def samples(kind, geo, seed):
    """(n_seg, seg_len) fp32 block.  mol: uniform in [-1, 1] with exact +1, -1, +0 and -0 sprinkled in (the first and
    last sample of every fold included).  raw / mu: class values, the 512 of them in the first fold's unfaded part."""
    rs = np.random.RandomState(seed)
    shape = (geo.n_seg, geo.seg_len)
    if kind == "mol":
        x = rs.uniform(-1, 1, shape).astype(F32)
        flat = x.reshape(-1)
        for v in (1.0, -1.0, 0.0, -0.0):
            flat[rs.choice(flat.size, max(1, flat.size // 40), replace=False)] = F32(v)
        x[:, 0], x[:, -1] = F32(1), F32(-1)
        x[0, 1], x[-1, 2] = F32(-0.0), F32(0.0)
        assert np.signbit(x[x == 0]).any() and (~np.signbit(x[x == 0])).any()
        return x
    lbl = rs.randint(0, N, shape)
    lo = geo.overlap
    mid = lbl[:, lo:geo.seg_len - lo].reshape(-1)
    assert mid.size >= N
    mid[:N] = rs.permutation(N)
    lbl[:, lo:geo.seg_len - lo] = mid.reshape(geo.n_seg, -1)
    return labels_to_samples(lbl)


def device_epilogue(m, x, geo, batched, wave_len, mu_law, override=None):
    """cabi.epilogue on x with m's tables; `override` (a dict) replaces call arguments (refusals).  Returns the
    waveform."""
    dev = torch.device("cuda", 0)
    tabs = m._epilogue_tables(geo, batched, mu_law, dev)
    p = lambda t: 0 if t is None else t.data_ptr()
    d = torch.as_tensor(x, device=dev)
    wav = torch.full((wave_len,), float("nan"), dtype=torch.float64, device=dev)
    kw = dict(samples=d.data_ptr(), n_seg=x.shape[0], seg_len=x.shape[1], seg_stride=geo.seg_stride, overlap=geo.overlap,
              fade_in=p(tabs["fade_in"]), fade_out=p(tabs["fade_out"]), mu_table=p(tabs["mu"]), n_classes=m.n_classes,
              tail=p(tabs["tail"]), tail_len=20 * m.hop_length, wave_len=wave_len, wav=wav.data_ptr(),
              stream=torch.cuda.current_stream(dev).cuda_stream)
    kw.update(override or {})
    cabi.epilogue(**kw)
    torch.cuda.synchronize(dev)
    out = wav.cpu().numpy()
    assert not np.isnan(out).any(), "waveform left unwritten"
    return out


def host_epilogue(m, x, geo, batched, wave_len, mu_law):
    return m._epilogue(x.astype(np.float64), geo, batched, wave_len, mu_law)


def oracle_epilogue(m, x, geo, batched, wave_len, mu_law):
    return O.epilogue(x, batched=batched, target=geo.target, overlap=geo.overlap, wave_len=wave_len,
                      hop_length=m.hop_length, mode="RAW", mu_law=mu_law, n_classes=N)


def grid_span():
    """Samples one pass of wrnn_epilogue's capped grid covers on this device (grid_stride_blocks: 8 blocks per SM)."""
    return 8 * torch.cuda.get_device_properties(0).multi_processor_count * 256


# (id, kind, batched, n_seg, target, overlap, hop, crop); seg_len of an unbatched case in `target`; n_seg None: the
# fewest folds whose wave spans more than three passes of the capped grid
CASES = [
    ("one-fold", "mol", True, 1, 700, 275, 3, 0),
    ("two-folds-overlap-2", "mol", True, 2, 300, 2, 9, 37),
    ("target-1-overlap-1", "mol", True, 40, 1, 1, 1, 0),
    ("target-below-odd-overlap", "mol", True, 40, 2, 3, 1, 7),
    ("target-below-overlap-276", "mol", True, 3, 100, 276, 8, 0),
    ("fade-out-is-the-wave", "mol", True, 5, 10, 3, 3, 8),
    ("overlap-275", "mol", True, 4, 5000, 275, 200, 1),
    ("three-grid-passes", "mol", True, None, 22000, 550, 275, 3),
    ("unbatched", "mol", False, 1, 6000, 0, 256, 100),
    ("raw-labels", "raw", True, 40, 200, 50, 300, 5),
    ("raw-labels-mu-law", "mu", True, 40, 200, 50, 300, 5),
    ("raw-labels-mu-law-unbatched", "mu", False, 1, 6000, 0, 200, 0),
    ("raw-labels-mu-law-overlap-1", "mu", True, 40, 20, 1, 1, 0),
]


@pytest.mark.parametrize("name,kind,batched,n_seg,target,overlap,hop,crop", CASES, ids=[c[0] for c in CASES])
def test_device_epilogue(name, kind, batched, n_seg, target, overlap, hop, crop):
    m = model(hop)
    if n_seg is None:
        n_seg = 3 * grid_span() // (target + overlap) + 2
    geo = geometry(batched, n_seg, target, overlap, seg_len=target)
    full = (geo.n_seg - 1) * geo.seg_stride + geo.seg_len
    wave_len = full - crop
    tail_len = 20 * hop
    assert tail_len <= wave_len
    if name == "fade-out-is-the-wave":
        assert tail_len == wave_len
    if name == "three-grid-passes":
        assert wave_len > 3 * grid_span()
    mu_law = kind == "mu"
    x = samples(kind, geo, seed=len(name))
    if kind != "mol":
        got = np.rint((x.astype(np.float64) + 1) * (N - 1) / 2)
        assert set(got[:, geo.overlap:geo.seg_len - geo.overlap].reshape(-1).astype(int)) == set(range(N))
    dev = device_epilogue(m, x, geo, batched, wave_len, mu_law)
    host = host_epilogue(m, x, geo, batched, wave_len, mu_law)
    ref = oracle_epilogue(m, x, geo, batched, wave_len, mu_law)
    assert dev.shape == host.shape == ref.shape == (wave_len,)
    assert np.array_equal(dev, host), ("device != host", int((dev != host).sum()))
    table_ulps = 0
    if mu_law:
        # the 512-entry table the device read against the oracle's expansion of the same class values
        xk = labels_to_samples(np.arange(N)).astype(np.float64)
        table = m._epilogue_tables(geo, batched, True, torch.device("cuda", 0))["mu"].cpu().numpy()
        pw = np.array([float(N) ** abs(v) for v in xk])
        d = np.abs(table - O.decode_mu_law(xk, N))
        assert (d <= np.spacing(pw) / (N - 1)).all()
        table_ulps = int((d > 0).sum())
        # each output sample sums at most two expanded values (each within 1 ulp of its power / 511) times weights
        # <= 1, with at most three roundings of its own
        bound = 2 * np.spacing(float(N)) / (N - 1) + 3 * np.spacing(np.abs(ref))
        off = dev != ref
        assert (np.abs(dev - ref)[off] <= bound[off]).all(), float(np.abs(dev - ref).max())
        n_off = int(off.sum())
    else:
        assert np.array_equal(dev, ref), ("device != oracle", int((dev != ref).sum()), float(np.abs(dev - ref).max()))
        n_off = 0
    print(f"epilogue {name}: {'batched' if batched else 'unbatched'} n_seg {geo.n_seg} target {geo.target} overlap "
          f"{geo.overlap} wave {wave_len} of {full} (fade-out {tail_len}): bit-exact vs host; vs oracle "
          f"{'bit-exact' if not n_off else f'{n_off} samples within 1 ulp of the mu-law power'}"
          f"{f'; mu-law table entries 1 ulp from the oracle {table_ulps}' if mu_law else ''}")


def test_epilogue_refusals_leave_the_next_call_exact():
    """Each argument wrnn_epilogue refuses, with its message; the valid call after each one is still bit-exact."""
    m = model(3)
    geo = geometry(True, 6, 100, 5)
    x = samples("mu", geo, seed=3)
    full = (geo.n_seg - 1) * geo.seg_stride + geo.seg_len
    want = host_epilogue(m, x, geo, True, full - 2, True)
    refusals = [
        ("overlap windows must not intersect", dict(overlap=geo.seg_len // 2 + 1)),
        ("wave_len exceeds the unfolded length", dict(wave_len=full + 1)),
        ("tail_len must be in (0, wave_len]", dict(tail_len=full - 1)),
        ("tail_len must be in (0, wave_len]", dict(tail_len=0)),
        ("fade tables are required when overlap > 0", dict(fade_in=0)),
        ("fade tables are required when overlap > 0", dict(fade_out=0)),
        ("wrnn_epilogue: n_classes", dict(n_classes=1)),
    ]
    for msg, override in refusals:
        with pytest.raises(cabi.EngineError, match=re.escape(msg)):
            device_epilogue(m, x, geo, True, full - 2, True, override)
        assert np.array_equal(device_epilogue(m, x, geo, True, full - 2, True), want), msg
