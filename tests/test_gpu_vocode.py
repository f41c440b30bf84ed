"""Vocoding a mel through the C ABI alone (wrnn_attach_upsampler / wrnn_conditioning_frames / wrnn_vocode): the
conditioning network on the device against torch's in float64, and the whole call against the public generate()."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import helpers
from wavernn_b200 import cabi

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
ROOT = helpers.GOLDEN.parent.parent
TARGET, OVERLAP = 2200, 220             # short folds, as smoke() uses


@pytest.fixture(scope="module")
def lib():
    if not cabi.is_built():
        import __graft_entry__ as g
        g.build()
    return cabi.load()


def _engine(model, precision="fp16", engine="auto"):
    eng = cabi.Engine(model.hot_state(), n_classes=model.n_classes, mode=model.mode, precision=precision, engine=engine)
    eng.attach_upsampler(model.state_dict())
    return eng


def _stream():
    return torch.cuda.current_stream(DEV).cuda_stream


def _frames(eng, mel):
    """The library's mel_frames, aux_frames and up_taps for mel (80, T) numpy."""
    T = mel.shape[1]
    d = torch.as_tensor(mel, dtype=torch.float32, device=DEV).contiguous()
    mf = torch.full((T + 4, 80), float("nan"), device=DEV)
    af = torch.full((T, 128), float("nan"), device=DEV)
    tp = torch.full((eng.hop_length, 5), float("nan"), device=DEV)
    eng.conditioning_frames(mel=d.data_ptr(), T=T, mel_frames=mf.data_ptr(), aux_frames=af.data_ptr(), up_taps=tp.data_ptr(),
                            stream=_stream())
    torch.cuda.synchronize(DEV)
    eng.check()
    return mf, af, tp


def _vocode(eng, mel, **kw):
    T = mel.shape[1]
    d = torch.as_tensor(mel, dtype=torch.float32, device=DEV).contiguous()
    wav = torch.full(((T - 1) * eng.hop_length,), float("nan"), dtype=torch.float64, device=DEV)
    eng.vocode(mel=d.data_ptr(), T=T, wav=wav.data_ptr(), stream=_stream(), **kw)
    torch.cuda.synchronize(DEV)
    eng.check()
    return wav.cpu().numpy()


def _randomise_batch_norms(m, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for mod in m.upsample.resnet.modules():
            if isinstance(mod, torch.nn.BatchNorm1d):
                mod.weight.uniform_(0.5, 1.5, generator=g)
                mod.bias.uniform_(-0.3, 0.3, generator=g)
                mod.running_mean.uniform_(-0.5, 0.5, generator=g)
                mod.running_var.uniform_(0.2, 2.0, generator=g)


def _mu_table(lib, n):
    mu = np.empty(n)
    assert lib.wrnn_debug_epilogue_tables(0, 1, n, 275, None, None, mu.ctypes.data, None) == 0
    return mu


# -------------------------------------------------------------------------------------------------- conditioning
def test_mel_frames_are_the_padded_mel(lib):
    m = helpers.make_model(0, "MOL")
    eng = _engine(m)
    for T in (21, 37, 200):
        mel = helpers.make_mel(T, seed=T)
        mf, _, _ = _frames(eng, mel[0].numpy())
        assert torch.equal(mf.cpu(), F.pad(mel, (2, 2))[0].T.contiguous()), T


def _aux_errors(eng, net, mel):
    """max |library - float64| and max |torch fp32 CPU - float64| of MelResNet's output on mel (80, T)."""
    mp = F.pad(torch.from_numpy(mel)[None], (2, 2))
    with torch.no_grad():
        t32 = net.float()(mp)[0].T.numpy().astype(np.float64)
        ref = net.double()(mp.double())[0].T.numpy()
        net.float()
    _, af, _ = _frames(eng, mel)
    return np.abs(af.cpu().numpy() - ref).max(), np.abs(t32 - ref).max()


@pytest.mark.parametrize("weights", ["random", "checkpoint"])
def test_aux_frames_against_float64(lib, weights):
    m = helpers.make_model(0, "MOL")
    if weights == "checkpoint":
        m.load_state_dict(helpers.pretrained_state_dict())
        mels = helpers.tacotron_mels() + [helpers.make_mel(T, seed=T)[0].numpy() for T in (21, 37, 200)]
    else:
        _randomise_batch_norms(m, 7)
        mels = [helpers.make_mel(T, seed=T)[0].numpy() for T in (21, 37, 64, 65, 200, 801)]
    net = m.upsample.resnet.eval()
    eng = _engine(m)
    worst = 0.0
    for mel in mels:
        e_lib, e_torch = _aux_errors(eng, net, mel)
        print(f"aux_frames {weights} T={mel.shape[1]}: library {e_lib:.3e}, torch fp32 CPU {e_torch:.3e} (vs float64)")
        assert e_lib <= 4 * e_torch, (mel.shape, e_lib, e_torch)
        worst = max(worst, e_lib / e_torch)
    print(f"aux_frames {weights}: worst ratio library / torch = {worst:.2f}")


def test_up_taps_match_upsample_taps(lib):
    m = helpers.make_model(0, "MOL")
    _, _, tp = _frames(_engine(m), helpers.make_mel(21)[0].numpy())
    ref = m.upsample_taps(torch.device("cpu"))
    assert (tp.cpu() - ref).abs().max().item() <= 2.0 ** -20 * ref.abs().max().item()


# -------------------------------------------------------------------------------------------------- vs generate()
def _patched_generate(model, eng, lib, mel, batched, target, overlap, mu_law):
    """generate(gen_rng='philox') with the library's aux_frames and taps in place of torch's (and, under mu_law, the
    library's mu-law table: numpy's np.power may differ from the C library's pow in the last bit, test_vocode_abi.py)."""
    _, af, tp = _frames(eng, mel)
    model.upsample_taps(DEV)                  # sets _taps_exact, read by _kernel_conditioning_ok
    resnet = model.upsample.resnet

    class Frames(torch.nn.Module):
        def forward(self, x):
            return af.T[None].contiguous()
    model.upsample.resnet = Frames()
    model.upsample_taps = lambda device: tp
    tables = model._epilogue_tables

    def lib_tables(geo, b, mu, device):
        t = dict(tables(geo, b, mu, device))
        if mu:
            t["mu"] = torch.from_numpy(_mu_table(lib, model.n_classes)).to(device)
        return t
    model._epilogue_tables = lib_tables
    try:
        return model.generate(torch.from_numpy(mel)[None], None, batched, target, overlap, mu_law)
    finally:
        model.upsample.resnet = resnet
        del model.upsample_taps, model._epilogue_tables


CASES = [  # mode, precision, gen_engine, batched, mu_law, T, target, overlap
    ("MOL", "fp16", "auto", True, False, 26, TARGET, OVERLAP),
    ("MOL", "fp16", "tcgen05", False, False, 26, TARGET, OVERLAP),
    ("MOL", "bf16", "tcgen05", True, False, 37, TARGET, OVERLAP),
    ("MOL", "fp16", "stream", True, False, 26, TARGET, OVERLAP),
    ("MOL", "bf16", "stream", False, False, 21, TARGET, OVERLAP),
    ("MOL", "fp16", "auto", True, False, 110, 100, 10),          # 274 folds: auto picks the stream engine
    ("RAW", "fp16", "auto", True, True, 26, TARGET, OVERLAP),
    ("RAW", "fp16", "tcgen05", True, False, 26, TARGET, OVERLAP),
    ("RAW", "bf16", "tcgen05", False, True, 21, TARGET, OVERLAP),
    ("RAW", "fp16", "stream", True, True, 37, TARGET, OVERLAP),
    ("RAW", "bf16", "stream", True, False, 26, TARGET, OVERLAP),
    ("RAW", "fp16", "auto", True, False, 110, 100, 10),
]


@pytest.mark.parametrize("mode,precision,gen_engine,batched,mu_law,T,target,overlap", CASES)
def test_vocode_equals_public_generate_on_the_same_frames(lib, mode, precision, gen_engine, batched, mu_law, T, target, overlap):
    m = helpers.make_model(0, mode, device=DEV)
    m.gen_rng, m.gen_precision, m.gen_engine, m.gen_philox_seed = "philox", precision, gen_engine, 1234
    eng = _engine(m, precision, gen_engine)
    mel = helpers.make_mel(T, seed=T)[0].numpy()
    want = _patched_generate(m, eng, lib, mel, batched, target, overlap, mu_law)
    got = _vocode(eng, mel, batched=batched, target=target, overlap=overlap, mu_law=mu_law, philox_seed=1234)
    print(f"{mode} {precision} {gen_engine} batched={batched} mu_law={mu_law}: engine {eng.name} vs {m.gen_stats['engine']}")
    assert eng.name == m.gen_stats["engine"]
    if gen_engine == "auto" and T == 110:
        assert ("stream" in eng.name) == (mode == "MOL")
    assert got.shape == want.shape and np.array_equal(got, want)


@pytest.mark.parametrize("mode,precision,batched", [("MOL", "fp32", True), ("RAW", "fp32", False), ("MOL", "bf16", True)])
def test_simt_handles_vocode_the_expanded_rows(lib, mode, precision, batched):
    """A SIMT handle takes per-sample rows: wrnn_vocode == Engine.generate on the rows expand_conditioning makes from the
    library's frames, then the device epilogue, bit for bit."""
    from wavernn_b200.sharding import fold_geometry, unbatched_geometry
    m = helpers.make_model(0, mode)
    eng = _engine(m, precision, "simt")
    T, seed = 26, 77
    mel = helpers.make_mel(T, seed=5)[0].numpy()
    got = _vocode(eng, mel, batched=batched, target=TARGET, overlap=OVERLAP, philox_seed=seed)
    mf, af, tp = _frames(eng, mel)
    L = T * 275
    geo = fold_geometry(L, TARGET, OVERLAP) if batched else unbatched_geometry(L)
    m_up = torch.empty(L, 80, device=DEV)
    aux = torch.empty(L, 128, device=DEV)
    cabi.expand_conditioning(mel_frames=mf.data_ptr(), aux_frames=af.data_ptr(), up_taps=tp.data_ptr(), hop=275, row_lo=0,
                             n_rows=L, mels_up=m_up.data_ptr(), aux=aux.data_ptr(), stream=_stream())
    out = torch.empty(geo.n_seg, geo.seg_len, device=DEV)
    eng.generate(mels_up=m_up.data_ptr(), aux=aux.data_ptr(), L=L, n_seg=geo.n_seg, seg_len=geo.seg_len,
                 seg_stride=geo.seg_stride, out=out.data_ptr(), philox_seed=seed, stream=_stream())
    tabs = m._epilogue_tables(geo, batched, False, DEV)
    wav = torch.empty((T - 1) * 275, dtype=torch.float64, device=DEV)
    p = lambda t: 0 if t is None else t.data_ptr()
    cabi.epilogue(samples=out.data_ptr(), n_seg=geo.n_seg, seg_len=geo.seg_len, seg_stride=geo.seg_stride,
                  overlap=geo.overlap if batched else 0, fade_in=p(tabs["fade_in"]), fade_out=p(tabs["fade_out"]), mu_table=0,
                  n_classes=m.n_classes, tail=p(tabs["tail"]), tail_len=20 * 275, wave_len=(T - 1) * 275, wav=wav.data_ptr(),
                  stream=_stream())
    torch.cuda.synchronize(DEV)
    eng.check()
    assert eng.name.startswith("simt")
    assert np.array_equal(got, wav.cpu().numpy())


@pytest.mark.parametrize("mode", ["MOL", "RAW"])
def test_vocode_against_unpatched_generate(lib, mode):
    """Against generate(gen_rng='philox') with torch's MelResNet on CUDA, random-init: MoL within DESIGN §5's 2e-2, RAW
    with >= 97 % identical samples (the generate_many criterion: within 1e-9, so that a mu-law table entry numpy's
    np.power rounds differently does not count as a different pick)."""
    m = helpers.make_model(0, mode, device=DEV)
    m.gen_rng, m.gen_philox_seed = "philox", 99
    eng = _engine(m)
    mel = helpers.make_mel(26, seed=3)[0].numpy()
    got = _vocode(eng, mel, target=TARGET, overlap=OVERLAP, mu_law=mode == "RAW", philox_seed=99)
    want = m.generate(torch.from_numpy(mel)[None], None, True, TARGET, OVERLAP, mode == "RAW")
    if mode == "MOL":
        err = np.abs(got - want).max()
        print(f"MoL vocode vs generate(): max |diff| = {err:.3e}")
        assert err <= 2e-2
    else:
        same = np.mean(np.abs(got - want) <= 1e-9)
        print(f"RAW vocode vs generate(): {100 * same:.2f} % identical samples ({100 * np.mean(got == want):.2f} % bit for bit)")
        assert same >= 0.97


@pytest.mark.parametrize("mode,batched", [("MOL", True), ("RAW", False)])
def test_host_entry_equals_device_entry(lib, mode, batched):
    m = helpers.make_model(0, mode)
    eng = _engine(m)
    mel = helpers.make_mel(30, seed=8)[0].numpy()
    kw = dict(batched=batched, target=TARGET, overlap=OVERLAP, mu_law=True, philox_seed=5)
    assert np.array_equal(eng.vocode_host(mel, **kw), _vocode(eng, mel, **kw))


@pytest.mark.parametrize("mode,precision", [("MOL", "fp16"), ("RAW", "fp32")])
def test_c_program_equals_vocode_host(lib, tmp_path, mode, precision):
    """examples/vocode_mel.c, run as its own process (no Python in it), on weight and mel files written here."""
    exe = ROOT / "wavernn_b200" / "wrnn_vocode_mel"
    assert exe.is_file(), "built by wavernn_b200/csrc/Makefile"
    m = helpers.make_model(0, mode)
    _randomise_batch_norms(m, 3)
    wdir = tmp_path / "weights"
    wdir.mkdir()
    for k, v in m.state_dict().items():
        v.detach().float().numpy().astype("<f4").tofile(wdir / f"{k}.f32")
    mel = helpers.make_mel(27, seed=2)[0].numpy()
    mel.astype("<f4").tofile(tmp_path / "mel.f32")
    env = {k: v for k, v in os.environ.items() if not k.startswith("PYTHON")}
    r = subprocess.run([str(exe), str(wdir), str(tmp_path / "mel.f32"), str(tmp_path / "wav.f64"), f"mode={mode}",
                        f"precision={precision}", f"target={TARGET}", f"overlap={OVERLAP}", "mu_law=1", "seed=31"],
                       capture_output=True, text=True, env=env, timeout=600)
    assert r.returncode == 0, r.stderr
    print(r.stdout.strip())
    got = np.fromfile(tmp_path / "wav.f64", dtype="<f8")
    eng = _engine(m, precision)
    want = eng.vocode_host(mel, target=TARGET, overlap=OVERLAP, mu_law=True, philox_seed=31)
    assert np.array_equal(got, want)


def test_refusals_leave_the_handle_usable(lib):
    m = helpers.make_model(0, "MOL")
    sd = m.state_dict()
    up = {k: v for k, v in sd.items() if k.startswith("upsample.")}
    bare = cabi.Engine(m.hot_state())
    mel = helpers.make_mel(26, seed=4)[0].numpy()
    with pytest.raises(cabi.EngineError, match="no upsampler attached"):
        bare.vocode_host(mel, target=TARGET, overlap=OVERLAP)
    bare.close()

    eng = _engine(m)
    kw = dict(target=TARGET, overlap=OVERLAP, philox_seed=2)
    first = eng.vocode_host(mel, **kw)

    def refused(match, fn, *a, **k):
        with pytest.raises(cabi.EngineError, match=match) as e:
            fn(*a, **k)
        assert e.value.code == cabi.WRNN_E_INVALID

    k = "upsample.resnet.layers.2.conv1.weight"
    refused(f"missing key: {k}", eng.attach_upsampler, {kk: v for kk, v in up.items() if kk != k})
    refused("unexpected key.*upsample.resnet.extra", eng.attach_upsampler, dict(up, **{"upsample.resnet.extra": up[k]}))
    refused("upsample.resnet.conv_out.bias has 127 elements", eng.attach_upsampler,
            dict(up, **{"upsample.resnet.conv_out.bias": up["upsample.resnet.conv_out.bias"][:127]}))
    refused("unsupported dims", eng.attach_upsampler, up, compute_dims=64)
    refused("unsupported dims", eng.attach_upsampler, up, res_out_dims=256)
    refused("5-tap", eng.attach_upsampler, up, pad=3)
    refused("5-tap", eng.attach_upsampler, up, hop_length=300)
    wide = dict(up, **{"upsample.up_layers.1.weight": torch.full((1, 1, 1, 3), 1 / 3.),
                       "upsample.up_layers.3.weight": torch.full((1, 1, 1, 11), 1 / 11.),
                       "upsample.up_layers.5.weight": torch.full((1, 1, 1, 111), 1 / 111.)})
    refused("5-tap", eng.attach_upsampler, wide, upsample_factors=(1, 5, 55))
    refused("T must be >= 21", eng.vocode_host, mel[:, :20], **kw)
    refused("target > 0 and overlap > 0", eng.vocode_host, mel, target=0, overlap=OVERLAP)
    refused("target > 0 and overlap > 0", eng.vocode_host, mel, target=TARGET, overlap=0)
    assert np.array_equal(eng.vocode_host(mel, **kw), first)
    assert np.array_equal(eng.vocode_host(mel, batched=False, overlap=0, target=0), eng.vocode_host(mel, batched=False))
    job = cabi.WrnnVocodeJob(None, 26, 1, TARGET, OVERLAP, 0, 0, None)
    assert lib.wrnn_vocode(eng._h, ctypes.byref(job), None) == cabi.WRNN_E_INVALID
    assert np.array_equal(eng.vocode_host(mel, **kw), first)
