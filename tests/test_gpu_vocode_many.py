"""A batch of mels through the C ABI as one job (wrnn_vocode_many / wrnn_vocode_many_host): every utterance's waveform
against its own wrnn_vocode call on the same handle, bit for bit, on every engine; one engine job per batch; the AUTO
routing by the batch's fold count; the refusals."""
import ctypes
import math
import os
import subprocess

import numpy as np
import pytest
import torch

import helpers
from wavernn_b200 import cabi
from wavernn_b200.sharding import fold_geometry

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
ROOT = helpers.GOLDEN.parent.parent
TARGET, OVERLAP = 2200, 220
TS = (26, 21, 40, 33)                    # frames of the utterances of a batch (different lengths)
SEEDS = (11, 2 ** 63 + 5, 0, 977)


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


def _mels(Ts, seed=0):
    return [helpers.make_mel(T, seed=seed + 100 * i + T)[0].numpy() for i, T in enumerate(Ts)]


def _folds(Ts, batched, target, overlap):
    return sum(fold_geometry(T * 275, target, overlap).n_seg for T in Ts) if batched else len(Ts)


def _singles(eng, mels, seeds, **kw):
    return [eng.vocode_host(m, philox_seed=s, **kw) for m, s in zip(mels, seeds)]


CASES = [  # mode, precision, engine, batched, mu_law
    ("MOL", "fp16", "tcgen05", True, False),
    ("MOL", "bf16", "tcgen05", False, False),
    ("RAW", "fp16", "tcgen05", True, True),
    ("RAW", "bf16", "tcgen05", False, False),
    ("MOL", "fp16", "stream", True, False),
    ("MOL", "bf16", "stream", False, False),
    ("RAW", "fp16", "stream", True, False),
    ("RAW", "bf16", "stream", False, True),
    ("MOL", "fp32", "simt", True, False),
    ("RAW", "fp32", "simt", False, True),
    ("MOL", "bf16", "simt", False, False),
    ("RAW", "bf16", "simt", True, True),
]


@pytest.mark.parametrize("mode,precision,engine,batched,mu_law", CASES)
def test_batch_equals_single_calls(lib, mode, precision, engine, batched, mu_law):
    m = helpers.make_model(0, mode)
    eng = _engine(m, precision, engine)
    mels = _mels(TS)
    kw = dict(batched=batched, target=TARGET, overlap=OVERLAP, mu_law=mu_law)
    want = _singles(eng, mels, SEEDS, **kw)
    n0 = eng.launch_count
    got = eng.vocode_many_host(mels, SEEDS, **kw)
    launches = eng.launch_count - n0
    folds = _folds(TS, batched, TARGET, OVERLAP)
    print(f"{mode} {precision} {engine} batched={batched} mu_law={mu_law}: {folds} folds, {launches} launches ({eng.name})")
    assert ("stream" in eng.name) == (engine == "stream") and eng.name.startswith("simt" if engine == "simt" else "tcgen05")
    if engine == "tcgen05":
        assert launches == math.ceil(folds / 64)
    elif engine == "stream":
        assert launches == 1
    for i, (g, w) in enumerate(zip(got, want)):
        assert g.shape == w.shape == ((TS[i] - 1) * 275,) and np.array_equal(g, w), i


@pytest.mark.parametrize("mode", ["MOL", "RAW"])
def test_tcgen05_batch_across_tiles(lib, mode):
    """Hundreds of folds: one utterance's folds straddle two tile-launches of 64."""
    m = helpers.make_model(0, mode)
    eng = _engine(m, "fp16", "tcgen05")
    Ts, seeds = (40, 37, 64), (3, 4, 5)
    mels = _mels(Ts, 7)
    kw = dict(target=100, overlap=10, mu_law=True)
    want = _singles(eng, mels, seeds, **kw)
    n0 = eng.launch_count
    got = eng.vocode_many_host(mels, seeds, **kw)
    folds = _folds(Ts, True, 100, 10)
    assert folds > 128 and fold_geometry(40 * 275, 100, 10).n_seg % 64 != 0
    assert eng.launch_count - n0 == math.ceil(folds / 64)
    for g, w in zip(got, want):
        assert np.array_equal(g, w)


def test_stream_batch_in_another_form(lib, monkeypatch):
    """The stream engine's form (folds per CTA, cluster) depends on the fold count; each fold's draws do not."""
    m = helpers.make_model(0, "MOL")
    eng = _engine(m, "fp16", "stream")
    mels = _mels(TS, 3)
    kw = dict(target=TARGET, overlap=OVERLAP)
    monkeypatch.setenv("WRNN_STREAM_NF", "16")
    monkeypatch.setenv("WRNN_STREAM_CL", "4")
    want = _singles(eng, mels, SEEDS, **kw)
    monkeypatch.setenv("WRNN_STREAM_NF", "32")
    monkeypatch.setenv("WRNN_STREAM_CL", "1")
    got = eng.vocode_many_host(mels, SEEDS, **kw)
    for g, w in zip(got, want):
        assert np.array_equal(g, w)


def test_seeds_and_order(lib):
    m = helpers.make_model(0, "MOL")
    eng = _engine(m, "fp16", "tcgen05")
    a, b = _mels((30, 24), 9)
    kw = dict(target=TARGET, overlap=OVERLAP)
    w = eng.vocode_many_host([a, a, a, b], [8, 8, 9, 8], **kw)
    assert np.array_equal(w[0], w[1])                     # same mel, same seed
    assert not np.array_equal(w[0], w[2])                 # same mel, another seed
    assert np.array_equal(w[0], eng.vocode_host(a, philox_seed=8, **kw))
    perm = [3, 0, 2, 1]
    mels, seeds = [a, a, a, b], [8, 8, 9, 8]
    p = eng.vocode_many_host([mels[i] for i in perm], [seeds[i] for i in perm], **kw)
    for k, i in enumerate(perm):
        assert np.array_equal(p[k], w[i])


def test_auto_routes_by_total_folds(lib):
    """An AUTO MoL batch of >= 257 folds goes to the stream engine, whose waveforms equal single calls on a stream
    handle bit for bit (the utterances alone would be served by the persistent engine)."""
    m = helpers.make_model(0, "MOL")
    auto, stream = _engine(m, "fp16", "auto"), _engine(m, "fp16", "stream")
    Ts, seeds = (40, 30, 36), (1, 2, 3)
    kw = dict(target=100, overlap=10)
    assert _folds(Ts, True, 100, 10) >= 257 and all(_folds([T], True, 100, 10) < 257 for T in Ts)
    mels = _mels(Ts, 5)
    got = auto.vocode_many_host(mels, seeds, **kw)
    assert "stream" in auto.name
    want = _singles(stream, mels, seeds, **kw)
    for g, w in zip(got, want):
        assert np.array_equal(g, w)


@pytest.mark.parametrize("mode,batched", [("MOL", True), ("RAW", False)])
def test_host_entry_equals_device_entry(lib, mode, batched):
    m = helpers.make_model(0, mode)
    eng = _engine(m)
    mels = _mels(TS, 2)
    kw = dict(batched=batched, target=TARGET, overlap=OVERLAP, mu_law=True)
    want = eng.vocode_many_host(mels, SEEDS, **kw)
    d_mels = [torch.as_tensor(x, device=DEV).contiguous() for x in mels]
    d_wavs = [torch.full(((x.shape[1] - 1) * 275,), float("nan"), dtype=torch.float64, device=DEV) for x in mels]
    eng.vocode_many(mels=[t.data_ptr() for t in d_mels], Ts=[x.shape[1] for x in mels], seeds=SEEDS,
                    wavs=[t.data_ptr() for t in d_wavs], stream=torch.cuda.current_stream(DEV).cuda_stream, **kw)
    torch.cuda.synchronize(DEV)
    eng.check()
    for g, w in zip(d_wavs, want):
        assert np.array_equal(g.cpu().numpy(), w)


def test_c_program_with_three_pairs(lib, tmp_path):
    exe = ROOT / "wavernn_b200" / "wrnn_vocode_mel"
    assert exe.is_file(), "built by wavernn_b200/csrc/Makefile"
    m = helpers.make_model(0, "MOL")
    wdir = tmp_path / "weights"
    wdir.mkdir()
    for k, v in m.state_dict().items():
        v.detach().float().numpy().astype("<f4").tofile(wdir / f"{k}.f32")
    mels = _mels((27, 22, 35), 4)
    args = []
    for i, mel in enumerate(mels):
        mel.astype("<f4").tofile(tmp_path / f"mel{i}.f32")
        args += [str(tmp_path / f"mel{i}.f32"), str(tmp_path / f"wav{i}.f64")]
    env = {k: v for k, v in os.environ.items() if not k.startswith("PYTHON")}
    r = subprocess.run([str(exe), str(wdir), *args, "mode=MOL", f"target={TARGET}", f"overlap={OVERLAP}", "seed=40"],
                       capture_output=True, text=True, env=env, timeout=600)
    assert r.returncode == 0, r.stderr
    print(r.stdout.strip())
    want = _engine(m).vocode_many_host(mels, [40, 41, 42], target=TARGET, overlap=OVERLAP)
    for i, w in enumerate(want):
        assert np.array_equal(np.fromfile(tmp_path / f"wav{i}.f64", dtype="<f8"), w)


def test_refusals_leave_the_handle_usable(lib):
    m = helpers.make_model(0, "MOL")
    bare = cabi.Engine(m.hot_state())
    mels = _mels(TS, 6)
    with pytest.raises(cabi.EngineError, match="no upsampler attached"):
        bare.vocode_many_host(mels, SEEDS)
    bare.close()

    eng = _engine(m, "fp16", "tcgen05")
    kw = dict(target=TARGET, overlap=OVERLAP)
    first = eng.vocode_many_host(mels, SEEDS, **kw)

    def refused(match, *a, **k):
        with pytest.raises(cabi.EngineError, match=match) as e:
            eng.vocode_many_host(*a, **k)
        assert e.value.code == cabi.WRNN_E_INVALID
    refused("utterance 2: T must be >= 21", mels[:2] + [mels[2][:, :20]] + mels[3:], SEEDS, **kw)
    refused("target > 0 and overlap > 0", mels, SEEDS, target=0, overlap=OVERLAP)
    refused("target > 0 and overlap > 0", mels, SEEDS, target=TARGET, overlap=0)
    refused("1 to 65535 utterances", [], [], **kw)
    b, keep = cabi.vocode_batch([(0x1000, 26, 0, 0x1000), (0, 26, 0, 0x1000)], target=TARGET, overlap=OVERLAP)
    assert lib.wrnn_vocode_many(eng._h, ctypes.byref(b), None) == cabi.WRNN_E_INVALID
    assert b"utterance 1: mel and wav are required" in lib.wrnn_last_error()
    del keep
    again = eng.vocode_many_host(mels, SEEDS, **kw)
    for g, w in zip(again, first):
        assert np.array_equal(g, w)
