"""The frame-rate conditioning kernels and the vocode paths at upsampling geometries other than (5, 5, 11) / 275.

The library serves any geometry whose interpolation cascade fits the 5-tap table (pad 2, factors whose product is the
hop, an impulse response within +-2 frames).  The hop enters the FRAMES staging of both engines (the persistent small
tile advances (frame, phase) row by row, the BIG tile and the stream engine divide per row), the conditioning pre-pass,
the C vocode path (T * hop rows, the 20-hop fade-out, the 4 * hop gap rows of a batch) and generate() /
generate_many().  Here, at hop 1 (1,), 3 (3,), 200 (5, 5, 8), 256 (4, 8, 8) and 600 (600,) (the pre-pass also at 8):

  - every FRAMES kernel (8 persistent, 16 stream) on the jobs of tests/kernel_jobs.py made at that hop, with the checks
    of tests/test_gpu_instantiations.py (logits within LOGIT_TOL of the emulation, samples, FRAMES == pre-pass rows,
    BIG == small tiles, cluster == one-CTA form);
  - the pre-pass against the float64 rows; up_taps against upsample_taps; aux_frames against the float64 MelResNet at
    0, 1 and 3 residual blocks;
  - wrnn_vocode against the public generate() on the same frames (persistent, stream, auto and SIMT handles), and
    wrnn_vocode_many against one call per utterance; against unpatched generate() at the criteria of test_gpu_vocode.py;
  - generate()'s frame-rate conditioning against the materialised torch path, and generate_many() against sequential
    generate() calls.
Run on a GPU: pytest -m gpu tests/test_gpu_geometries.py -s (one line per kernel and hop)."""
import math

import numpy as np
import pytest
import torch

import helpers
import kernel_jobs as K
from test_gpu_instantiations import PERSISTENT, STREAM, Matrix, check_persistent_kernel, check_pre_pass, check_stream_kernel
from test_gpu_vocode import _aux_errors, _frames, _patched_generate, _randomise_batch_norms, _vocode
from wavernn_b200 import cabi
from wavernn_b200.sharding import fold_geometry, unbatched_geometry

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
HOPS = K.KERNEL_HOPS                      # 1, 3, 200, 256, 600


@pytest.fixture(scope="module")
def lib():
    if not cabi.is_built():
        import __graft_entry__ as g
        g.build()
    return cabi.load()


def _model(hop, mode="MOL", device="cpu", **kw):
    return K.geometry_model(hop, mode, **kw).to(device)


def _engine(model, precision="fp16", engine="auto"):
    eng = cabi.Engine(model.hot_state(), n_classes=model.n_classes, mode=model.mode, precision=precision, engine=engine)
    up = model.upsample
    eng.attach_upsampler(model.state_dict(), res_blocks=len(up.resnet.layers),
                         upsample_factors=tuple(s.x_scale for s in up.up_layers[0::2]), hop_length=model.hop_length)
    return eng


def _scaled(hop):
    """(T, target, overlap) of the vocode cases: the reference's 26 frames with 2200 / 220 at hop 275, scaled to the hop,
    so that a batched job has 3 folds, the last one padded."""
    T, target, overlap = 26, 8 * hop, max(2, 4 * hop // 5)
    geo = fold_geometry(T * hop, target, overlap)
    assert geo.n_seg >= 3 and geo.padded_len > T * hop and 20 * hop < (T - 1) * hop
    return T, target, overlap


# ------------------------------------------------------------------------------------------------ the kernel matrix
class HopMatrix(Matrix):
    """test_gpu_instantiations.Matrix with jobs made at `hop`; the models and engines (independent of the hop) shared."""

    def __init__(self, shared, hop):
        super().__init__()
        self.models, self.engines = shared.models, shared.engines
        self.hop, self.taps = hop, K.geometry_taps(hop)

    def job(self, n, head, tables):
        if (n, head, tables) not in self.jobs:
            self.jobs[(n, head, tables)] = K.make_job(n, head, self.taps, tables, hop=self.hop)
        return self.jobs[(n, head, tables)]


@pytest.fixture(scope="module")
def matrix():
    """matrix(hop): the jobs, emulations and runs of one hop at a time (the tests run hop by hop)."""
    shared, cur = Matrix(), {}

    def at(hop):
        if hop not in cur:
            cur.clear()
            cur[hop] = HopMatrix(shared, hop)
        return cur[hop]
    yield at
    shared.close()


TC = [(hop, p, h, big) for hop in HOPS for p, h, fr, big in PERSISTENT if fr]
SK = [(hop, p, h, nf, cl) for hop in HOPS for p, h, fr, nf, cl in STREAM if fr]


@pytest.mark.parametrize("hop,precision,head,big", TC, ids=[f"hop{hop}-tc-{p}-{h}-{'big' if b else 'small'}" for hop, p, h, b in TC])
def test_persistent_frames_kernel_at_other_hops(matrix, hop, precision, head, big):
    check_persistent_kernel(matrix(hop), precision, head, True, big, tag=f"hop {hop}: ")


@pytest.mark.parametrize("hop,precision,head,nf,cl", SK, ids=[f"hop{hop}-stream-{p}-{h}-{nf}x{cl}" for hop, p, h, nf, cl in SK])
def test_stream_frames_kernel_at_other_hops(matrix, hop, precision, head, nf, cl):
    check_stream_kernel(matrix(hop), precision, head, True, nf, cl, tag=f"hop {hop}: ")


@pytest.mark.parametrize("hop", [1, 3, 8, 200, 256, 600])
def test_conditioning_pre_pass_at_other_hops(hop):
    """test_conditioning_pre_pass_against_the_float64_rows at `hop`, with enough frames for more than two passes of
    the capped grid."""
    n_sm = torch.cuda.get_device_properties(DEV).multi_processor_count
    check_pre_pass(K.geometry_taps(hop), hop, max(80, (2 * 8 * 8 * n_sm + 57) // hop + 2))


# ------------------------------------------------------------------------------------------ the conditioning network
@pytest.mark.parametrize("hop", HOPS)
def test_up_taps_at_other_geometries(lib, hop):
    m = _model(hop)
    _, _, tp = _frames(_engine(m), helpers.make_mel(21)[0].numpy())
    ref = m.upsample_taps(torch.device("cpu"))
    err = (tp.cpu() - ref).abs().max().item()
    print(f"hop {hop}: up_taps max |library - upsample_taps| {err:.2e} (bound {2.0 ** -20 * ref.abs().max().item():.2e})")
    assert err <= 2.0 ** -20 * ref.abs().max().item()


@pytest.mark.parametrize("res_blocks", [0, 1, 3])
@pytest.mark.parametrize("hop", HOPS)
def test_aux_frames_at_other_geometries(lib, hop, res_blocks):
    """test_aux_frames_against_float64's criterion (4 x torch's fp32 CPU error) with other residual block counts, T on
    both sides of the 64-frame CTA tile."""
    m = _model(hop, res_blocks=res_blocks)
    _randomise_batch_norms(m, 7 + res_blocks)
    net = m.upsample.resnet.eval()
    eng = _engine(m)
    worst = 0.0
    for T in (21, 64, 65, 130):
        e_lib, e_torch = _aux_errors(eng, net, helpers.make_mel(T, seed=T)[0].numpy())
        assert e_lib <= 4 * e_torch, (T, e_lib, e_torch)
        worst = max(worst, e_lib / e_torch)
    print(f"hop {hop} res_blocks {res_blocks}: aux_frames worst ratio library / torch fp32 CPU error = {worst:.2f} (bound 4)")


# ------------------------------------------------------------------------------------------------------ the C vocode
VOCODE = [  # mode, precision, gen_engine, batched, mu_law
    ("MOL", "fp16", "auto", True, False),
    ("MOL", "bf16", "tcgen05", False, False),
    ("MOL", "fp16", "stream", True, False),
    ("RAW", "fp16", "tcgen05", True, True),
    ("RAW", "bf16", "stream", False, True),
    ("RAW", "fp16", "auto", True, False),
]


@pytest.mark.parametrize("mode,precision,gen_engine,batched,mu_law", VOCODE)
@pytest.mark.parametrize("hop", HOPS)
def test_vocode_equals_public_generate_at_other_geometries(lib, hop, mode, precision, gen_engine, batched, mu_law):
    T, target, overlap = _scaled(hop)
    m = _model(hop, mode, DEV)
    m.gen_rng, m.gen_precision, m.gen_engine, m.gen_philox_seed = "philox", precision, gen_engine, 1234
    eng = _engine(m, precision, gen_engine)
    mel = helpers.make_mel(T, seed=T + hop)[0].numpy()
    want = _patched_generate(m, eng, lib, mel, batched, target, overlap, mu_law)
    assert m.gen_stats["conditioning"] == "kernel"
    got = _vocode(eng, mel, batched=batched, target=target, overlap=overlap, mu_law=mu_law, philox_seed=1234)
    print(f"hop {hop} {mode} {precision} {gen_engine} batched={batched} mu_law={mu_law}: engine {eng.name}, "
          f"{m.gen_stats['n_seg']} folds x {m.gen_stats['seg_len']} steps")
    assert eng.name == m.gen_stats["engine"] and ("stream" in eng.name) == (gen_engine == "stream")
    assert got.shape == want.shape == ((T - 1) * hop,) and np.array_equal(got, want)


@pytest.mark.parametrize("mode,precision", [("MOL", "fp32"), ("RAW", "bf16")])
@pytest.mark.parametrize("hop", HOPS)
def test_simt_handle_vocodes_the_expanded_rows_at_other_geometries(lib, hop, mode, precision):
    """test_simt_handles_vocode_the_expanded_rows at `hop`: wrnn_vocode on a SIMT handle == Engine.generate on the
    rows expand_conditioning makes from the library's frames, then the device epilogue, bit for bit."""
    T, target, overlap = _scaled(hop)
    m = _model(hop, mode)
    eng = _engine(m, precision, "simt")
    mel = helpers.make_mel(T, seed=5)[0].numpy()
    got = _vocode(eng, mel, target=target, overlap=overlap, philox_seed=77)
    mf, af, tp = _frames(eng, mel)
    L = T * hop
    geo = fold_geometry(L, target, overlap)
    m_up = torch.empty(L, 80, device=DEV)
    aux = torch.empty(L, 128, device=DEV)
    st = torch.cuda.current_stream(DEV).cuda_stream
    cabi.expand_conditioning(mel_frames=mf.data_ptr(), aux_frames=af.data_ptr(), up_taps=tp.data_ptr(), hop=hop, row_lo=0,
                             n_rows=L, mels_up=m_up.data_ptr(), aux=aux.data_ptr(), stream=st)
    out = torch.empty(geo.n_seg, geo.seg_len, device=DEV)
    eng.generate(mels_up=m_up.data_ptr(), aux=aux.data_ptr(), L=L, n_seg=geo.n_seg, seg_len=geo.seg_len,
                 seg_stride=geo.seg_stride, out=out.data_ptr(), philox_seed=77, stream=st)
    tabs = m._epilogue_tables(geo, True, False, DEV)
    wav = torch.empty((T - 1) * hop, dtype=torch.float64, device=DEV)
    cabi.epilogue(samples=out.data_ptr(), n_seg=geo.n_seg, seg_len=geo.seg_len, seg_stride=geo.seg_stride,
                  overlap=geo.overlap, fade_in=tabs["fade_in"].data_ptr(), fade_out=tabs["fade_out"].data_ptr(), mu_table=0,
                  n_classes=m.n_classes, tail=tabs["tail"].data_ptr(), tail_len=20 * hop, wave_len=(T - 1) * hop,
                  wav=wav.data_ptr(), stream=st)
    torch.cuda.synchronize(DEV)
    eng.check()
    assert eng.name.startswith("simt")
    assert np.array_equal(got, wav.cpu().numpy())


MANY = [  # mode, precision, engine, batched, mu_law
    ("MOL", "fp16", "tcgen05", True, False),
    ("RAW", "bf16", "tcgen05", False, True),
    ("MOL", "bf16", "stream", True, False),
    ("RAW", "fp16", "stream", True, True),
    ("MOL", "fp32", "simt", True, False),
]


@pytest.mark.parametrize("mode,precision,engine,batched,mu_law", MANY)
@pytest.mark.parametrize("hop", [3, 256])
def test_vocode_many_equals_single_calls_at_other_geometries(lib, hop, mode, precision, engine, batched, mu_law):
    """Utterances of different lengths: each one's padded last fold runs past its end over the 4 * hop gap rows that
    separate it from the next one in the batch's stream."""
    _, target, overlap = _scaled(hop)
    Ts, seeds = (26, 21, 40, 33), (11, 2 ** 63 + 5, 0, 977)
    assert all(fold_geometry(T * hop, target, overlap).padded_len > T * hop for T in Ts)
    m = _model(hop, mode)
    eng = _engine(m, precision, engine)
    mels = [helpers.make_mel(T, seed=100 * i + T)[0].numpy() for i, T in enumerate(Ts)]
    kw = dict(batched=batched, target=target, overlap=overlap, mu_law=mu_law)
    want = [eng.vocode_host(x, philox_seed=s, **kw) for x, s in zip(mels, seeds)]
    n0 = eng.launch_count
    got = eng.vocode_many_host(mels, seeds, **kw)
    folds = sum(fold_geometry(T * hop, target, overlap).n_seg for T in Ts) if batched else len(Ts)
    print(f"hop {hop} {mode} {precision} {engine} batched={batched}: {folds} folds, {eng.launch_count - n0} launches ({eng.name})")
    if engine == "tcgen05":
        assert eng.launch_count - n0 == math.ceil(folds / 64)
    for i, (g, w) in enumerate(zip(got, want)):
        assert g.shape == w.shape == ((Ts[i] - 1) * hop,) and np.array_equal(g, w), i


def _compare(mode, got, want, what):
    """MoL within DESIGN §5's 2e-2; RAW with >= 97 % of the samples within 1e-9."""
    if mode == "MOL":
        err = np.abs(got - want).max()
        print(f"{what}: MoL max |diff| = {err:.3e} (bound 2e-2)")
        assert err <= 2e-2
    else:
        same = np.mean(np.abs(got - want) <= 1e-9)
        print(f"{what}: RAW {100 * same:.2f} % identical samples (bound 97 %)")
        assert same >= 0.97


@pytest.mark.parametrize("mode", ["MOL", "RAW"])
@pytest.mark.parametrize("hop", HOPS)
def test_vocode_against_unpatched_generate_at_other_geometries(lib, hop, mode):
    T, target, overlap = _scaled(hop)
    m = _model(hop, mode, DEV)
    m.gen_rng, m.gen_philox_seed = "philox", 99
    eng = _engine(m)
    mel = helpers.make_mel(T, seed=3)[0].numpy()
    got = _vocode(eng, mel, target=target, overlap=overlap, mu_law=mode == "RAW", philox_seed=99)
    want = m.generate(torch.from_numpy(mel)[None], None, True, target, overlap, mode == "RAW")
    _compare(mode, got, want, f"hop {hop} vocode vs generate()")


# ------------------------------------------------------------------------------------------- generate / generate_many
@pytest.mark.parametrize("mode", ["MOL", "RAW"])
@pytest.mark.parametrize("hop", [3, 256])
def test_generate_kernel_conditioning_against_torch_at_other_geometries(hop, mode):
    """gen_conditioning='kernel' (rows formed by the library from the 5-tap table) against 'torch' (UpsampleNetwork's
    rows, the reference's upsample)."""
    T, target, overlap = _scaled(hop)
    m = _model(hop, mode, DEV)
    m.gen_rng, m.gen_philox_seed = "philox", 5
    mel = helpers.make_mel(T, seed=hop)
    wavs = {}
    for cond in ("kernel", "torch"):
        m.gen_conditioning = cond
        wavs[cond] = m.generate(mel, None, True, target, overlap, mode == "RAW")
        assert m.gen_stats["conditioning"] == cond
    _compare(mode, wavs["kernel"], wavs["torch"], f"hop {hop} generate() kernel vs torch conditioning")


@pytest.mark.parametrize("mode", ["MOL", "RAW"])
@pytest.mark.parametrize("hop", [3, 256])
def test_generate_many_equals_sequential_generate_calls_at_other_geometries(hop, mode):
    """test_generate_many_equals_sequential_generate_calls at `hop`, reference-compatible draws."""
    _, target, overlap = _scaled(hop)
    m = _model(hop, mode, DEV)
    mels = [helpers.make_mel(T, seed) for T, seed in ((30, 0), (26, 3), (41, 5), (22, 7))]
    torch.manual_seed(99)
    seq = [m.generate(x, None, True, target, overlap, mode == "RAW") for x in mels]
    assert m.gen_stats["conditioning"] == "kernel"
    torch.manual_seed(99)
    many = m.generate_many(mels, [None] * len(mels), target, overlap, mode == "RAW")
    assert m.gen_stats["utterances"] == 4
    for a, b in zip(seq, many):
        assert a.shape == b.shape
        np.testing.assert_allclose(b, a, rtol=0, atol=1e-6)
    print(f"hop {hop} {mode}: generate_many == sequential generate() within 1e-6, "
          f"max |diff| {max(np.abs(a - b).max() for a, b in zip(seq, many)):.1e}")
