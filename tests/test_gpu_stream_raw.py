"""The stream engine's 9-bit RAW head (wavernn_b200/csrc/wrnn_stream.cu, RAW = true): fc3 in four blocks of 128
classes, per-class Exp(1) draws keyed like the other engines, the pick reduced over warps, blocks and (cluster form)
ranks with ties to the lowest class.  Its step program and cluster protocol are checked on the CPU
(tests/test_stream_plan_raw.py); this file runs the four forms (16 / 32 folds per CTA x one CTA / a 4-CTA cluster) on
the GPU against the host restatement of the draws, the reference fixture, the persistent engine and each other.
Run on a GPU: pytest -m gpu."""
import numpy as np
import pytest
import torch

import helpers
from gpu_helpers import run_engine
from oracle import philox as P
from oracle import wavernn_oracle as O
from test_gpu_sampling import (OFFSET, SEED, SEG_FIRST, Runner, crafted, forced_inputs, inputs, kernel_picks,
                               raw_bias, raw_host_picks)

pytestmark = pytest.mark.gpu

STREAM_FORMS = ["stream-16x1", "stream-16x4", "stream-32x1", "stream-32x4"]


@pytest.fixture(scope="module")
def raw_model():
    return helpers.make_model(0, "RAW", "cuda")


@pytest.mark.parametrize("form", STREAM_FORMS)
def test_stream_raw_philox_draws_equal_the_restated_draws_and_host_picks(form, raw_model, monkeypatch):
    """Teacher-forced: a Philox run equals a run fed oracle/philox.raw_expo's draws as `expo`, samples and logits bit
    for bit, and its picks are the host's argmax over its logits and those draws wherever the margin exceeds 1e-5."""
    steps = 16
    with Runner(raw_model, form, monkeypatch) as run:
        B = run.n_seg
        m_up, aux = inputs(B, steps, 1)
        xf = forced_inputs(B, steps, 2)
        out, lg = run(m_up, aux, steps, x_force=xf)
        expo, _ = P.raw_expo(SEED, OFFSET, SEG_FIRST, B, steps)
        out_e, lg_e = run(m_up, aux, steps, x_force=xf, expo=expo)
        out_w, _ = run(m_up, aux, steps, x_force=xf, seg_first=0)           # other keys, other picks: not vacuous
    assert np.array_equal(out, out_e) and np.array_equal(lg, lg_e)
    assert not np.array_equal(out_w, out)
    want, margin = raw_host_picks(lg, expo)
    got = kernel_picks(out)
    clear = margin > 1e-5
    print(f"{form}: {got.size} RAW picks, {int((~clear).sum())} closer than 1e-5, {int((got != want)[clear].sum())} differ where clear")
    assert clear.mean() >= 0.99 and np.array_equal(got[clear], want[clear])


@pytest.mark.parametrize("form", STREAM_FORMS)
def test_stream_raw_zero_draw_of_seed_220_picks_as_the_host_does(form, raw_model, monkeypatch):
    """Seed 220's word at (fold 0, step 29, class 489) maps to u01 = 1; the clamped draw makes 489 the host's pick."""
    steps, seed = 32, 220
    with Runner(raw_model, form, monkeypatch) as run:
        B = run.n_seg
        expo, words = P.raw_expo(seed, 0, 0, B, steps)
        assert words[29, 0, 489] >> 8 == 0xFFFFFF
        m_up, aux = inputs(B, steps, 6)
        out, lg = run(m_up, aux, steps, seg_first=0, seed=seed, offset=0, x_force=forced_inputs(B, steps, 7))
    want, margin = raw_host_picks(lg, expo)
    got = kernel_picks(out)
    print(f"{form}: at (fold 0, step 29) host {want[29, 0]} (margin {margin[29, 0]:.3f}), kernel {got[29, 0]}")
    assert want[29, 0] == 489 and got[29, 0] == 489 and margin[29, 0] > 1e-3
    clear = margin > 1e-5
    assert np.array_equal(got[clear], want[clear])


@pytest.mark.parametrize("form", STREAM_FORMS)
def test_stream_raw_exact_ties_go_to_the_lowest_class(form, monkeypatch):
    """fc3 weight 0 (logits = bias bitwise), equal bias maxima in different 128-class blocks and different warps of a
    block, every draw 1: the lowest tied class wins, across warps, blocks and cluster ranks."""
    steps = 8
    bias = raw_bias()
    bias[:] = np.minimum(bias, 1.0)
    tied = [77, 90, 200, 300, 511]                       # two warps of block 0, then blocks 1, 2, 3
    bias[tied] = 2.0
    model = crafted("RAW", bias)
    with Runner(model, form, monkeypatch) as run:
        B = run.n_seg
        m_up, aux = inputs(B, steps, 4)
        out, lg = run(m_up, aux, steps, expo=np.ones((steps, B, 512), np.float32))
    assert (lg == bias).all()
    assert (kernel_picks(out) == 77).all()
    bias[77] = 1.0                                        # the next tie: blocks 0 (row 90) vs 1, 2, 3
    model = crafted("RAW", bias)
    with Runner(model, form, monkeypatch) as run:
        out, _ = run(m_up, aux, steps, expo=np.ones((steps, B, 512), np.float32))
    assert (kernel_picks(out) == 90).all()


@pytest.fixture(scope="module")
def fixture_job(raw_model):
    g = helpers.load_golden("raw_batched.npz")
    expo = helpers.replay_expo(1234, 3300, 3, 512)
    if not np.array_equal(expo[:8], g["expo_head"]):
        pytest.skip("torch exponential_() stream differs on this host")
    sd = helpers.state_numpy(raw_model)
    m_up, aux = O.upsample_network(sd, O.pad_time(helpers.make_mel(30, 0)[0].numpy().T, 2).T, pad=2)
    return dict(g=g, expo=expo, m_up=m_up, aux=aux)


def test_stream_raw_teacher_forced_against_the_reference_fixture_and_the_persistent_engine(raw_model, fixture_job):
    g, J = fixture_job["g"], fixture_job
    kw = dict(n_seg=3, seg_len=3300, seg_stride=3025, expo=J["expo"], x_force=g["raw"].T.copy(), want_logits=True)
    lgs = {}
    for prec, frac, tol in (("fp16", 0.97, 5e-3), ("bf16", 0.90, 5e-2)):
        out, lg, name = run_engine(raw_model, J["m_up"], J["aux"], precision=prec, engine="stream", **kw)
        assert name.startswith(f"tcgen05-stream") and name.endswith(prec)
        same, lerr = (out == g["raw"]).mean(), np.abs(lg[:64] - g["logits"]).max()
        print(f"{name} RAW teacher-forced vs reference: identical picks {same:.4f}, logits err {lerr:.3e}")
        assert same >= frac and lerr <= tol
        lgs[prec] = lg
    _, lg_t, tname = run_engine(raw_model, J["m_up"], J["aux"], precision="fp16", engine="tcgen05", steps=600, **kw)
    d = np.abs(lgs["fp16"][:600] - lg_t).max()
    print(f"stream vs {tname} teacher-forced logits (600 steps): {d:.3e}")
    assert d <= 1e-3


@pytest.mark.parametrize("n_seg", [3, 17, 50, 70])
def test_stream_raw_cluster_form_equals_single_cta_form(n_seg, raw_model, monkeypatch):
    """Same MMAs in the same order, and a max with a lowest-class tie-break: the cluster form's samples and logits are
    those of the one-CTA form bit for bit (ragged tiles, zero-padded tail, free-running Philox)."""
    rs = np.random.RandomState(n_seg)
    seg_len, stride = 60, 40
    L = (n_seg - 1) * stride + 45
    m_up, aux = rs.rand(L, 80).astype(np.float32), rs.randn(L, 128).astype(np.float32)
    outs = {}
    for nf in ("16", "32"):
        for cl in ("1", "4"):
            monkeypatch.setenv("WRNN_STREAM_NF", nf); monkeypatch.setenv("WRNN_STREAM_CL", cl)
            out, lg, name = run_engine(raw_model, m_up, aux, n_seg=n_seg, seg_len=seg_len, seg_stride=stride, want_logits=True,
                                       engine="stream", philox_seed=(7 << 32) | 3, seg_first=5)
            assert name == ("tcgen05-stream-x4-fp16" if cl == "4" else "tcgen05-stream-fp16"), name
            outs[(nf, cl)] = (out, lg)
    for nf in ("16", "32"):
        assert np.array_equal(outs[(nf, "1")][0], outs[(nf, "4")][0]) and np.array_equal(outs[(nf, "1")][1], outs[(nf, "4")][1]), nf
    labels = (outs[("16", "1")][0] + 1) * 255.5
    assert np.abs(labels - np.rint(labels)).max() <= 1e-3 and labels.std() > 10


def test_stream_raw_cfg5_4096_folds_shard_invariance_and_the_persistent_engine(raw_model):
    """T = 172,034 frames -> 4096 RAW folds, first 48 steps, frame-rate conditioning, Philox: any sub-range generated on
    its own with its seg_first (with or without fold tables) reproduces its rows bit for bit; one 64-fold tile on the
    persistent engine picks as the stream engine does, teacher-forced, wherever the margin exceeds 1e-3."""
    from wavernn_b200 import cabi
    from wavernn_b200.sharding import fold_geometry
    dev = torch.device("cuda")
    T, hop, steps, seed = 172_034, 275, 48, 11
    geo = fold_geometry(T * hop, 11_000, 550)
    assert geo.n_seg == 4096
    torch.manual_seed(0)
    mel = torch.rand(1, 80, T, device=dev)
    with torch.no_grad():
        mp = torch.nn.functional.pad(mel, (2, 2))
        mel_fr = mp[0].transpose(0, 1).contiguous()
        aux_fr = raw_model.eval().upsample.resnet(mp)[0].transpose(0, 1).contiguous()
        taps = raw_model.upsample_taps(dev)

    def run(eng, f0, n, tables=False, x_force=None):
        row0 = (torch.arange(f0, f0 + n, device=dev, dtype=torch.int64) * geo.seg_stride).contiguous()
        end = torch.full_like(row0, T * hop)
        out = torch.full((n, steps), float("nan"), device=dev)
        lg = torch.full((steps, n, 512), float("nan"), device=dev) if x_force is not None else None
        xf = torch.as_tensor(x_force, device=dev) if x_force is not None else None
        eng.generate(mels_up=0, aux=0, L=T * hop, n_seg=n, seg_len=geo.seg_len, seg_stride=geo.seg_stride, out=out.data_ptr(),
                     seg_first=f0, steps=steps, philox_seed=seed, fold_row0=row0.data_ptr() if tables else 0,
                     fold_row_end=end.data_ptr() if tables else 0, mel_frames=mel_fr.data_ptr(), aux_frames=aux_fr.data_ptr(),
                     up_taps=taps.data_ptr(), hop=hop, x_force=xf.data_ptr() if xf is not None else 0,
                     logits_out=lg.data_ptr() if lg is not None else 0, stream=torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        eng.check()
        return (out.cpu().numpy(), lg.cpu().numpy()) if lg is not None else out.cpu().numpy()

    eng = cabi.Engine(raw_model.hot_state(), n_classes=512, mode="RAW", precision="fp16", engine="stream", device=0)
    big = run(eng, 0, 4096)
    assert eng.name == "tcgen05-stream-fp16" and eng.grid_ctas == 128 and eng.launch_count == 1
    labels = (big + 1) * 255.5
    assert np.isfinite(big).all() and np.abs(labels - np.rint(labels)).max() <= 1e-3 and labels.std() > 10
    for f0, n in ((0, 64), (64 * 37, 64), (4096 - 64, 64), (512 * 5, 512), (4000, 96)):
        assert np.array_equal(run(eng, f0, n), big[f0:f0 + n]), (f0, n)
    assert np.array_equal(run(eng, 512 * 3, 512, tables=True), big[512 * 3:512 * 4])
    f0 = 64 * 37
    xf = forced_inputs(64, steps, 9)
    out_s, lg_s = run(eng, f0, 64, x_force=xf)
    eng.close()
    tc = cabi.Engine(raw_model.hot_state(), n_classes=512, mode="RAW", precision="fp16", engine="tcgen05", device=0)
    out_t, _ = run(tc, f0, 64, x_force=xf)
    tc.close()
    expo, _ = P.raw_expo(seed, 0, f0, 64, steps)
    _, margin = raw_host_picks(lg_s, expo)
    clear = margin > 1e-3
    agree = (kernel_picks(out_s) == kernel_picks(out_t))
    print(f"cfg5 RAW tile 37, teacher-forced: stream vs persistent picks agree {agree.mean():.4f}, {agree[clear].mean():.4f} where clear")
    assert clear.mean() >= 0.99 and agree[clear].all()


def test_stream_raw_public_generate_generate_many_and_auto_routing(raw_model, fixture_job):
    g = fixture_job["g"]
    mel = helpers.make_mel(30, 0)
    model = raw_model
    model.gen_engine = "stream"
    try:
        torch.manual_seed(1234)
        wav = model.generate(mel, None, True, 2750, 275, True)
        assert model.gen_stats["engine"].startswith("tcgen05-stream") and model.gen_stats["conditioning"] == "kernel"
        assert wav.shape == g["wav"].shape and np.isfinite(wav).all() and np.abs(wav).max() <= 1.0
        same = (wav == g["wav"]).mean()
        print(f"stream engine RAW generate() vs reference wav: identical samples {same:.4f}, max {np.abs(wav - g['wav']).max():.3e}")
        # random-init model: every free-running pick equals the reference's, as on the persistent engine (measured on an
        # H100: identical waveform); a single near-tie resolved the other way would make this exact check fail
        assert np.array_equal(wav, g["wav"])
        mels = [helpers.make_mel(T, seed) for T, seed in ((30, 0), (24, 3), (35, 5))]
        for rng in ("torch", "philox"):
            model.gen_rng = rng
            torch.manual_seed(99)
            seq = [model.generate(m, None, True, 2750, 275, True) for m in mels]
            torch.manual_seed(99)
            many = model.generate_many(mels, [None] * 3, 2750, 275, True)
            assert model.gen_stats["engine"].startswith("tcgen05-stream")
            # torch draws: per-utterance streams, every utterance exact; Philox: keyed by global fold, utterance 0 exact
            for a, b in (zip(seq, many) if rng == "torch" else [(seq[0], many[0])]):
                assert np.array_equal(a, b), rng
    finally:
        model.gen_engine, model.gen_rng = "auto", "torch"
    # AUTO keeps RAW jobs on the persistent engine, however many folds
    rs = np.random.RandomState(0)
    n_seg, seg_len, stride = 300, 8, 10
    L = (n_seg - 1) * stride + 10
    m_up, aux = rs.rand(L, 80).astype(np.float32), rs.randn(L, 128).astype(np.float32)
    _, name = run_engine(model, m_up, aux, n_seg=n_seg, seg_len=seg_len, seg_stride=stride, engine="auto", philox_seed=3)
    assert name == "tcgen05-fp16", name
