"""The STREAM engine (wavernn_b200/csrc/wrnn_stream.cu: activation-stationary, weights streamed from L2, one independent
CTA per 16/32 folds) through the C ABI, against the engine-arithmetic emulation, the reference fixtures and the
persistent tcgen05 engine.  Its packing and step program are checked on the CPU (tests/test_stream_plan.py); this file
covers what only hardware can: descriptors, wgmma fragments, the mbarrier protocol, the ring.  Run on a GPU: pytest -m gpu."""
import numpy as np
import pytest
import torch

import helpers
from gpu_helpers import run_engine
from oracle import contract as C
from oracle import wavernn_oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def mol():
    model = helpers.make_model(0, "MOL", "cuda")
    sd = helpers.state_numpy(model)
    mel_p = O.pad_time(helpers.make_mel(30, 0)[0].numpy().T, 2).T
    m_up, aux = O.upsample_network(sd, mel_p, pad=2)
    return dict(model=model, sd=sd, w=O.hot_weights(sd), m_up=m_up, aux=aux, U=helpers.replay_uniforms(1234, 3300, 3),
                g=helpers.load_golden("mol_batched.npz"), kw=dict(n_seg=3, seg_len=3300, seg_stride=3025))


@pytest.mark.parametrize("precision", ["fp16", "bf16"])
def test_stream_engine_matches_emulation_and_reference_fixture(mol, precision):
    out, lg, name = run_engine(mol["model"], mol["m_up"], mol["aux"], uniforms=mol["U"], want_logits=True,
                               precision=precision, engine="stream", **mol["kw"])
    assert name in (f"tcgen05-stream-{precision}", f"tcgen05-stream-x4-{precision}")
    emu, lemu = C.generate_segments(mol["w"], mol["m_up"], mol["aux"], uniforms=mol["U"], precision=precision,
                                    want_logits=True, **mol["kw"])
    d_emu, d_ref = np.abs(out - emu), np.abs(out - mol["g"]["raw"])
    print(f"{name}: vs emulation max {d_emu.max():.3e} (logits {np.abs(lg - lemu).max():.3e}); vs reference max {d_ref.max():.3e}")
    tol_emu, tol_ref = (1e-3, 2e-2) if precision == "fp16" else (2e-2, 5e-2)
    assert np.isfinite(out).all() and d_emu.max() <= tol_emu and d_ref.max() <= tol_ref


def test_stream_engine_teacher_forced_logits_vs_reference_and_persistent_engine(mol):
    g = mol["g"]
    kw = dict(uniforms=mol["U"], x_force=g["raw"].T.copy(), want_logits=True, steps=600, **mol["kw"])
    _, lg_s, name = run_engine(mol["model"], mol["m_up"], mol["aux"], engine="stream", **kw)
    _, lg_t, _ = run_engine(mol["model"], mol["m_up"], mol["aux"], engine="tcgen05", **kw)
    print(f"{name} teacher-forced logits: vs reference {np.abs(lg_s - g['logits']).max():.3e}, vs persistent engine {np.abs(lg_s - lg_t).max():.3e}")
    assert np.abs(lg_s - g["logits"]).max() <= 5e-3 and np.abs(lg_s - lg_t).max() <= 1e-3


@pytest.mark.parametrize("n_seg", [1, 16, 17, 50])
def test_stream_engine_tiles_of_16_ragged_and_zero_padded_tail(n_seg):
    model = helpers.make_model(3, "MOL", "cuda")
    w = O.hot_weights(helpers.state_numpy(model))
    rs = np.random.RandomState(n_seg)
    seg_len, stride = 120, 80
    L = (n_seg - 1) * stride + 70                          # the last fold runs 50 rows past the end
    m_up, aux = rs.rand(L, 80).astype(np.float32), rs.randn(L, 128).astype(np.float32)
    U = helpers.replay_uniforms(5, seg_len, n_seg)
    kw = dict(n_seg=n_seg, seg_len=seg_len, seg_stride=stride, uniforms=U)
    out, lg, name = run_engine(model, m_up, aux, engine="stream", want_logits=True, **kw)
    emu, lemu = C.generate_segments(w, m_up, aux, precision="fp16", want_logits=True, **kw)
    print(f"{name} n_seg={n_seg}: vs emulation {np.abs(out - emu).max():.3e}, logits {np.abs(lg - lemu).max():.3e}")
    assert name.startswith("tcgen05-stream") and np.abs(out - emu).max() <= 1e-3 and np.abs(lg - lemu).max() <= 1e-3


def test_stream_engine_tiles_of_32_and_auto_selection():
    """More folds than 16 per SM: tiles of 32 folds (the other instantiation).  ENGINE_AUTO must route the job to the
    stream engine, and every tile must equal the same folds generated on their own (fold-keyed Philox)."""
    model = helpers.make_model(0, "MOL", "cuda")
    w = O.hot_weights(helpers.state_numpy(model))
    rs = np.random.RandomState(2)
    n_seg, seg_len, stride = 2400, 24, 10
    L = (n_seg - 1) * stride + 20
    m_up, aux = rs.rand(L, 80).astype(np.float32), rs.randn(L, 128).astype(np.float32)
    kw = dict(seg_len=seg_len, seg_stride=stride, philox_seed=11)
    big, name = run_engine(model, m_up, aux, n_seg=n_seg, engine="auto", **kw)
    assert name.startswith("tcgen05-stream") and np.isfinite(big).all() and np.abs(big).max() <= 1.0 and big.std() > 0.05
    for f0, n in ((0, 16), (640, 7), (2368, 32)):          # tiles of 16 (small jobs) reproduce rows of the 32-fold tiles
        off = f0 * stride
        part, pname = run_engine(model, m_up[off:], aux[off:], n_seg=n, seg_first=f0, engine="stream", **kw)
        assert np.array_equal(part, big[f0:f0 + n]), (f0, n)
    # against the emulation with explicit draws (32-fold tiles, 75 CTAs)
    U = helpers.replay_uniforms(3, seg_len, n_seg)
    out, _ = run_engine(model, m_up, aux, n_seg=n_seg, seg_len=seg_len, seg_stride=stride, uniforms=U, engine="stream")
    emu = C.generate_segments(w, m_up, aux, n_seg=n_seg, seg_len=seg_len, seg_stride=stride, uniforms=U, precision="fp16")
    print(f"{name} 2400 folds in tiles of 32: vs emulation {np.abs(out - emu).max():.3e}")
    assert np.abs(out - emu).max() <= 1e-3
    # few folds stay on the persistent engine
    _, name = run_engine(model, m_up, aux, n_seg=19, engine="auto", **kw)
    assert name == "tcgen05-fp16"


def test_stream_engine_public_generate_frames_and_materialised_conditioning(mol):
    """WaveRNN.generate(gen_engine='stream'): rows formed by the staging warps from frame-rate tensors (default) ==
    materialised UpsampleNetwork rows, and both track the reference wav."""
    model, g = mol["model"], mol["g"]
    mel = helpers.make_mel(30, 0)
    model.gen_engine = "stream"
    wavs = {}
    try:
        for mode in ("kernel", "torch"):
            model.gen_conditioning = mode
            torch.manual_seed(1234)
            wavs[mode] = model.generate(mel, None, True, 2750, 275, False)
            assert model.gen_stats["engine"].startswith("tcgen05-stream") and model.gen_stats["conditioning"] == mode
    finally:
        model.gen_engine, model.gen_conditioning = "auto", "kernel"
    d = np.abs(wavs["kernel"] - wavs["torch"]).max()
    print("stream engine, frame-rate vs materialised conditioning:", d, "| vs reference wav", np.abs(wavs["kernel"] - g["wav"]).max())
    assert d <= 1e-4 and np.abs(wavs["kernel"] - g["wav"]).max() <= 2e-2


def test_stream_engine_generate_many_with_fold_tables(mol):
    """Several utterances in one job (per-fold windows): the stream engine on the job == one generate() per utterance."""
    model = mol["model"]
    mels = [helpers.make_mel(T, seed) for T, seed in ((30, 0), (26, 3), (41, 5))]
    model.gen_engine = "stream"
    try:
        torch.manual_seed(99)
        seq = [model.generate(m, None, True, 2750, 275, False) for m in mels]
        torch.manual_seed(99)
        many = model.generate_many(mels, [None] * 3, 2750, 275, False)
        assert model.gen_stats["engine"].startswith("tcgen05-stream")
    finally:
        model.gen_engine = "auto"
    for a, b in zip(seq, many):
        np.testing.assert_allclose(b, a, rtol=0, atol=1e-6)


def test_stream_engine_trained_checkpoint_teacher_forced():
    g = helpers.load_golden("trained_tacotron.npz")
    model = helpers.make_model(0, "MOL", "cpu")
    model.load_state_dict(helpers.pretrained_state_dict(), strict=False)
    model = model.to("cuda")
    sd = helpers.state_numpy(model)
    mel = helpers.tacotron_mels()[int(g["sentence"])]
    m_up, aux = O.upsample_network(sd, O.pad_time(mel.T, 2).T, pad=2)
    U = helpers.replay_uniforms(int(g["seed"]), 12100, 4)
    _, lg, name = run_engine(model, m_up, aux, uniforms=U, x_force=g["raw"].T.copy(), want_logits=True, steps=600,
                             engine="stream", n_seg=4, seg_len=12100, seg_stride=11550)
    e = np.abs(lg - g["logits"])
    print(f"{name} trained teacher-forced logits: max {e.max():.3e} p99.9 {np.quantile(e, 0.999):.3e} median {np.median(e):.3e}")
    assert e.max() <= 1e-1 and np.quantile(e, 0.999) <= 3e-2 and np.median(e) <= 1e-3


def test_stream_engine_cfg5_4096_folds_shard_invariance_and_agreement_with_the_persistent_engine():
    """BASELINE configs[4] at its full fold count (T = 172,034 frames -> 4096 folds; first 48 steps): frame-rate
    conditioning formed by the staging warps, 128 CTAs of 32 folds.  Size-independent properties: any shard / tile of
    the job generated on its own (other tile size, other seg_first) reproduces its rows bit for bit (fold-keyed Philox,
    fold-independent arithmetic), with or without fold tables; and the persistent tcgen05 engine -- different
    decomposition, same rounding contract -- agrees to accumulation-order noise."""
    from wavernn_b200 import cabi
    from wavernn_b200.sharding import fold_geometry
    model = helpers.make_model(0, "MOL", "cuda")
    dev = torch.device("cuda")
    T, hop, steps = 172_034, 275, 48
    geo = fold_geometry(T * hop, 11_000, 550)
    assert geo.n_seg == 4096
    torch.manual_seed(0)
    mel = torch.rand(1, 80, T, device=dev)
    with torch.no_grad():
        mp = torch.nn.functional.pad(mel, (2, 2))
        mel_fr = mp[0].transpose(0, 1).contiguous()
        aux_fr = model.eval().upsample.resnet(mp)[0].transpose(0, 1).contiguous()
        taps = model.upsample_taps(dev)

    def run(eng, f0, n, tables=False):
        row0 = (torch.arange(f0, f0 + n, device=dev, dtype=torch.int64) * geo.seg_stride).contiguous()
        end = torch.full_like(row0, T * hop)
        out = torch.full((n, steps), float("nan"), device=dev)
        eng.generate(mels_up=0, aux=0, L=T * hop, n_seg=n, seg_len=geo.seg_len, seg_stride=geo.seg_stride, out=out.data_ptr(),
                     seg_first=f0, steps=steps, philox_seed=11, fold_row0=row0.data_ptr() if tables else 0,
                     fold_row_end=end.data_ptr() if tables else 0, mel_frames=mel_fr.data_ptr(), aux_frames=aux_fr.data_ptr(),
                     up_taps=taps.data_ptr(), hop=hop, stream=torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        eng.check()
        return out.cpu().numpy()

    eng = cabi.Engine(model.hot_state(), n_classes=30, mode="MOL", precision="fp16", engine="stream", device=0)
    big = run(eng, 0, 4096)
    assert eng.name == "tcgen05-stream-fp16" and eng.grid_ctas == 128 and eng.launch_count == 1
    assert np.isfinite(big).all() and np.abs(big).max() <= 1.0 and big.std() > 0.05
    for f0, n in ((0, 64), (64 * 37, 64), (4096 - 64, 64), (512 * 5, 512), (4000, 96)):
        assert np.array_equal(run(eng, f0, n), big[f0:f0 + n]), (f0, n)
    assert np.array_equal(run(eng, 512 * 3, 512, tables=True), big[512 * 3:512 * 4])
    eng.close()
    tc = cabi.Engine(model.hot_state(), n_classes=30, mode="MOL", precision="fp16", engine="tcgen05", device=0)
    ref = run(tc, 64 * 37, 64)
    tc.close()
    d = np.abs(ref - big[64 * 37:64 * 38]).max()
    print("cfg5 fold tile 37: stream engine vs persistent engine:", d)
    assert d <= 1e-3


@pytest.mark.parametrize("n_seg", [3, 16, 17, 50, 70])
def test_stream_engine_cluster_form_equals_single_cta_form_and_the_emulation(n_seg, monkeypatch):
    """Cluster form (WRNN_STREAM_CL=4: four CTAs split the rows of every layer, operand blocks pushed into each other's
    shared memory over DSMEM, cluster-scope barriers) vs the one-CTA form on the same job: the same MMAs in the same
    order, so the samples must be IDENTICAL; both within the emulation's tolerance.  Tiles of 16 and 32 folds."""
    model = helpers.make_model(3, "MOL", "cuda")
    w = O.hot_weights(helpers.state_numpy(model))
    rs = np.random.RandomState(n_seg)
    seg_len, stride = 120, 80
    L = (n_seg - 1) * stride + 70
    m_up, aux = rs.rand(L, 80).astype(np.float32), rs.randn(L, 128).astype(np.float32)
    U = helpers.replay_uniforms(5, seg_len, n_seg)
    kw = dict(n_seg=n_seg, seg_len=seg_len, seg_stride=stride, uniforms=U, engine="stream", want_logits=True)
    emu, lemu = C.generate_segments(w, m_up, aux, precision="fp16", want_logits=True, n_seg=n_seg, seg_len=seg_len, seg_stride=stride, uniforms=U)
    outs = {}
    for nf in ("16", "32"):
        for cl in ("1", "4"):
            monkeypatch.setenv("WRNN_STREAM_NF", nf); monkeypatch.setenv("WRNN_STREAM_CL", cl)
            out, lg, name = run_engine(model, m_up, aux, **kw)
            assert name.startswith("tcgen05-stream-x4" if cl == "4" else "tcgen05-stream-fp16"), name
            outs[(nf, cl)] = (out, lg)
            assert np.abs(out - emu).max() <= 1e-3 and np.abs(lg - lemu).max() <= 1e-3, (nf, cl)
    for nf in ("16", "32"):
        assert np.array_equal(outs[(nf, "1")][0], outs[(nf, "4")][0]) and np.array_equal(outs[(nf, "1")][1], outs[(nf, "4")][1]), nf
    print(f"cluster form n_seg={n_seg}: identical to the one-CTA form; vs emulation {np.abs(outs[('16', '4')][0] - emu).max():.3e}")


def test_stream_engine_cluster_form_public_generate_and_trained_logits(mol, monkeypatch):
    """The cluster form through the public call (frame-rate conditioning, streamed draws) and on the trained checkpoint."""
    model, g = mol["model"], mol["g"]
    monkeypatch.setenv("WRNN_STREAM_CL", "4")
    mel = helpers.make_mel(30, 0)
    model.gen_engine = "stream"
    try:
        torch.manual_seed(1234)
        wav = model.generate(mel, None, True, 2750, 275, False)
        assert model.gen_stats["engine"].startswith("tcgen05-stream-x4")
    finally:
        model.gen_engine = "auto"
    print("cluster form generate() vs reference wav:", np.abs(wav - g["wav"]).max())
    assert np.abs(wav - g["wav"]).max() <= 2e-2
    gt = helpers.load_golden("trained_tacotron.npz")
    tm = helpers.make_model(0, "MOL", "cpu")
    tm.load_state_dict(helpers.pretrained_state_dict(), strict=False)
    tm = tm.to("cuda")
    sd = helpers.state_numpy(tm)
    m_up, aux = O.upsample_network(sd, O.pad_time(helpers.tacotron_mels()[int(gt["sentence"])].T, 2).T, pad=2)
    U = helpers.replay_uniforms(int(gt["seed"]), 12100, 4)
    _, lg, name = run_engine(tm, m_up, aux, uniforms=U, x_force=gt["raw"].T.copy(), want_logits=True, steps=600, engine="stream",
                             n_seg=4, seg_len=12100, seg_stride=11550)
    e = np.abs(lg - gt["logits"])
    print(f"{name} trained teacher-forced logits: max {e.max():.3e} median {np.median(e):.3e}")
    assert name.startswith("tcgen05-stream-x4") and e.max() <= 1e-1 and np.quantile(e, 0.999) <= 3e-2 and np.median(e) <= 1e-3
