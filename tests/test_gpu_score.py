"""wrnn_score and wrnn_score_many on the GPU: the per-sample training loss of the reference, teacher-forced.

  1. The same chains as generation: wrnn_score's logits_out is bit-identical to wrnn_generate's with the same x_force,
     on every scoring instantiation (persistent fp16 | bf16 x MoL | RAW x rows | FRAMES x small | BIG tile; stream fp16 |
     bf16 x rows | FRAMES x 16 | 32 folds x 1 | 4 CTAs, MoL; SIMT fp32 | fp16 | bf16 x MoL | RAW), on the jobs of
     tests/kernel_jobs.py (persistent also at 73 folds over two launches, SIMT at 73 folds in three tiles); rows of nll
     at and past `steps` stay untouched.
  2. The loss arithmetic: nll against tests/score_oracle.py evaluated on that run's own logits, within its tolerance.
  3. Against the reference: the SIMT fp32 engine against tests/golden/score_pins.npz (b) and (c), within bounds derived
     on the CPU (tests/test_score_abi.py).
  4. Mel level: wrnn_score_many equals, bit for bit, each utterance alone, wrnn_score fed wrnn_conditioning_frames'
     tensors, the host entry and the permuted batch, on fixed-engine handles; 70 recordings on a persistent handle (two
     launches) equal the host entry and, at both ends of each launch, themselves alone; an AUTO handle sends 257
     utterances to the stream engine.
  5. Quality on the H100: the shipped checkpoint on the Tacotron fixture at fp16 / bf16 on both tensor-core engines
     against SIMT fp32 (median, mean, share of samples moved by > 1 nat), pinned against the same statistics of the
     CPU emulation's logits at each precision.
Run on a GPU: pytest -m gpu -s tests/test_gpu_score.py"""
import os

import numpy as np
import pytest
import torch

import helpers
import kernel_jobs as K
import score_oracle as SO
from oracle import contract as C
from oracle import wavernn_oracle as O
from wavernn_b200 import cabi

pytestmark = pytest.mark.gpu

PRECISIONS, HEADS = ("fp16", "bf16"), ("MOL", "RAW")
# tile sizes: the last small tile, the first BIG tile, a 64-fold BIG tile then a 9-fold small one over two launches
TILES = {"small": K.SMALL_TILE, "big": K.SMALL_TILE + 1, "tiles": 73}
PERSISTENT = [(p, h, fr, size) for p in PRECISIONS for h in HEADS for fr in (False, True) for size in TILES]
STREAM = [(p, fr, nf, cl) for p in PRECISIONS for fr in (False, True) for nf in (16, 32) for cl in (1, 4)]
SIMT = [(p, h, n) for n in (K.SMALL_TILE, 73) for p in ("fp32", "fp16", "bf16") for h in HEADS]   # 73: three tiles
# SIMT fp32 against the reference's own loss (score_pins.npz (b), (c)): tests/test_score_abi.py asserts each is at least
# 4 x the largest gap between the fp32 CPU emulation + score_oracle and the fixture.
from test_score_abi import RAND_TOL, TRAINED_TOL  # noqa: E402


class State:
    def __init__(self):
        self.models, self.engines, self.jobs = {}, {}, {}

    def model(self, head):
        if head not in self.models:
            m = helpers.make_model(0, head)
            taps = m.upsample_taps(torch.device("cpu")).numpy()
            self.models[head] = (m.to("cuda"), taps)
        return self.models[head]

    def engine(self, kind, precision, head):
        key = (kind, precision, head)
        if key not in self.engines:
            m = self.model(head)[0]
            self.engines[key] = cabi.Engine(m.hot_state(), n_classes=m.n_classes, mode=head, precision=precision,
                                            engine=kind, device=0)
        return self.engines[key]

    def job(self, n, head, tables):
        if (n, head, tables) not in self.jobs:
            self.jobs[(n, head, tables)] = K.make_job(n, head, self.model(head)[1], tables)
        return self.jobs[(n, head, tables)]

    def close(self):
        for e in self.engines.values():
            e.close()


@pytest.fixture(scope="module")
def st():
    s = State()
    yield s
    s.close()


def run(eng, job, frames, score, form=None):
    """The whole job on `eng`, generated (score=False) or scored.  Returns (samples or nll [SEG_LEN, n], logits)."""
    dev = torch.device("cuda", 0)
    n = job["n"]
    t = lambda x: None if x is None else torch.as_tensor(np.ascontiguousarray(x), device=dev)
    p = lambda x: 0 if x is None else x.data_ptr()
    row0, end = t(job["fold_row0"]), t(job["fold_row_end"])
    keep = []
    kw = dict(mels_up=0, aux=0, mel_frames=0, aux_frames=0, up_taps=0, hop=0)
    if frames:
        keep = [t(job["mel_frames"]), t(job["aux_frames"]), t(job["taps"])]
        kw.update(mel_frames=p(keep[0]), aux_frames=p(keep[1]), up_taps=p(keep[2]), hop=job["hop"])
        L = job["L"]
    else:
        keep = [t(job["m_up"]), t(job["aux"])]
        kw.update(mels_up=p(keep[0]), aux=p(keep[1]))
        L = job["L"] - job["row_lo"]
    nc = 30 if job["mode"] == "MOL" else 512
    lg = torch.full((K.STEPS, n, nc), float("nan"), device=dev)
    X = t(job["x_force"])
    saved = {v: os.environ.get(v) for v in ("WRNN_STREAM_NF", "WRNN_STREAM_CL")}
    if form is not None:
        os.environ["WRNN_STREAM_NF"], os.environ["WRNN_STREAM_CL"] = str(form[0]), str(form[1])
    s = torch.cuda.current_stream(dev).cuda_stream
    cond = cabi.COND_IN_KERNEL if frames and not job["tables"] else cabi.COND_AUTO
    try:
        if score:
            out = torch.full((K.SEG_LEN, n), float("nan"), device=dev)
            eng.score(L=L, n_seg=n, seg_len=K.SEG_LEN, seg_stride=K.STRIDE, seg_first=K.SEG_FIRST, steps=K.STEPS, x_force=p(X),
                      nll=p(out), logits_out=p(lg), fold_row0=p(row0), fold_row_end=p(end), cond_mode=cond, stream=s, **kw)
        else:
            out = torch.full((n, K.STEPS), float("nan"), device=dev)
            U, E = t(job["uniforms"]), t(job["expo"])
            eng.generate(L=L, n_seg=n, seg_len=K.SEG_LEN, seg_stride=K.STRIDE, out=p(out), seg_first=K.SEG_FIRST,
                         steps=K.STEPS, uniforms=p(U), expo=p(E), x_force=p(X), logits_out=p(lg), fold_row0=p(row0),
                         fold_row_end=p(end), cond_mode=cond, stream=s, **kw)
    finally:
        for v, old in saved.items():
            if old is None:
                os.environ.pop(v, None)
            else:
                os.environ[v] = old
    torch.cuda.synchronize(dev)
    eng.check()
    return out.cpu().numpy(), lg.cpu().numpy()


def check_scoring(eng, job, frames, form=None, what=""):
    _, lg_gen = run(eng, job, frames, False, form)
    nll, lg = run(eng, job, frames, True, form)
    assert np.array_equal(lg, lg_gen), f"{what}: scoring ran other chains than generation"
    assert np.isnan(nll[K.STEPS:]).all(), f"{what}: rows at and past `steps` were written"
    nll = nll[:K.STEPS]
    assert not np.isnan(nll).any()
    S, n, nc = lg.shape
    y = job["x_force"][:K.STEPS].reshape(-1)
    if job["mode"] == "MOL":
        want = SO.mol_loss(lg.reshape(-1, nc), y)
        tol, _ = SO.mol_loss_tolerance(lg.reshape(-1, nc), y)
    else:
        want = SO.raw_loss(lg.reshape(-1, nc), y)
        tol = SO.raw_loss_tolerance(lg.reshape(-1, nc))
    d = np.abs(nll.reshape(-1).astype(np.float64) - want)
    print(f"{what} [{eng.name}]: max |nll - oracle(own logits)| {d.max():.3e} (worst / tolerance {(d / tol).max():.3f})")
    i = int(np.argmax(d / tol))
    assert (d <= tol).all(), (what, float((d / tol).max()), "worst sample", i, float(y[i]), float(nll.reshape(-1)[i]), float(want[i]))


@pytest.mark.parametrize("precision,head,frames,size", PERSISTENT,
                         ids=[f"tc-{p}-{h}-{'frames' if fr else 'rows'}-{size}" for p, h, fr, size in PERSISTENT])
def test_persistent_scoring(st, precision, head, frames, size):
    eng = st.engine("tcgen05", precision, head)
    job = st.job(TILES[size], head, frames)
    n0 = eng.launch_count
    check_scoring(eng, job, frames, what=f"tc-{precision}-{head}-{'frames' if frames else 'rows'}-{size}")
    assert eng.name.startswith("tcgen05-")
    assert eng.launch_count - n0 == 2 * -(-TILES[size] // 64)          # generation and scoring, 64 folds per launch


@pytest.mark.parametrize("precision,frames,nf,cl", STREAM,
                         ids=[f"stream-{p}-{'frames' if fr else 'rows'}-nf{nf}-cl{cl}" for p, fr, nf, cl in STREAM])
def test_stream_scoring(st, precision, frames, nf, cl):
    eng = st.engine("stream", precision, "MOL")
    job = st.job(K.STREAM_FOLDS[nf], "MOL", frames)
    check_scoring(eng, job, frames, form=(nf, cl), what=f"stream-{precision}-nf{nf}-cl{cl}-{'frames' if frames else 'rows'}")
    assert ("-x4-" in eng.name) == (cl == 4)


@pytest.mark.parametrize("precision,head,n", SIMT, ids=[f"simt-{p}-{h}" + ("-tiles" if n == 73 else "") for p, h, n in SIMT])
def test_simt_scoring(st, precision, head, n):
    eng = st.engine("simt", precision, head)
    check_scoring(eng, st.job(n, head, False), False, what=f"simt-{precision}-{head}" + ("-tiles" if n == 73 else ""))


def test_stream_refuses_raw_scoring(st):
    m = st.model("RAW")[0]
    eng = cabi.Engine(m.hot_state(), n_classes=512, mode="RAW", precision="fp16", engine="stream")
    try:
        job = st.job(K.STREAM_FOLDS[16], "RAW", False)
        with pytest.raises(cabi.EngineError, match="MoL head only"):
            run(eng, job, False, True)
        eng.attach_upsampler(m.state_dict())
        mel = np.random.RandomState(0).rand(80, 8).astype(np.float32)
        with pytest.raises(cabi.EngineError, match="MoL head only"):
            eng.score_many_host([mel], [np.zeros(100, np.float32)])
    finally:
        eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# against the reference
# ---------------------------------------------------------------------------------------------------------------------
def score_rows(model, m_up, aux, x, *, n_seg, seg_len, seg_stride, precision, engine, want_logits=False):
    """wrnn_score on materialised rows; x (n_seg, seg_len) targets.  Returns nll (n_seg, seg_len), the engine's name
    [, logits (seg_len * n_seg, 30)]."""
    dev = torch.device("cuda", 0)
    eng = cabi.Engine(model.hot_state(), n_classes=model.n_classes, mode=model.mode, precision=precision, engine=engine)
    try:
        t = lambda a: torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float32, device=dev)
        d_m, d_a, d_x = t(m_up), t(aux), t(np.asarray(x).T)
        nll = torch.full((seg_len, n_seg), float("nan"), device=dev)
        lg = torch.empty((seg_len, n_seg, 30), device=dev) if want_logits else None
        eng.score(mels_up=d_m.data_ptr(), aux=d_a.data_ptr(), L=m_up.shape[0], n_seg=n_seg, seg_len=seg_len, seg_stride=seg_stride,
                  x_force=d_x.data_ptr(), nll=nll.data_ptr(), logits_out=lg.data_ptr() if want_logits else 0,
                  stream=torch.cuda.current_stream(dev).cuda_stream)
        torch.cuda.synchronize(dev)
        eng.check()
        res = (nll.cpu().numpy().T, eng.name)
        return res + (lg.cpu().numpy().transpose(1, 0, 2).reshape(-1, 30),) if want_logits else res
    finally:
        eng.close()


@pytest.fixture(scope="module")
def trained():
    model = helpers.make_model(0, "MOL", "cpu")
    missing = model.load_state_dict(helpers.pretrained_state_dict(), strict=False)
    assert not missing.missing_keys and not missing.unexpected_keys
    sd = helpers.state_numpy(model)
    g = helpers.load_golden("trained_tacotron.npz")
    mel = helpers.tacotron_mels()[int(g["sentence"])]
    m_up, aux = O.upsample_network(sd, O.pad_time(mel.T, 2).T, pad=2)
    return dict(model=model.to("cuda"), sd=sd, g=g, m_up=m_up, aux=aux)


def test_simt_fp32_against_reference(trained):
    pins = helpers.load_golden("score_pins.npz")
    g = trained["g"]
    nll, name, lg = score_rows(trained["model"], trained["m_up"], trained["aux"], g["raw"], n_seg=4, seg_len=12100,
                               seg_stride=11550, precision="fp32", engine="simt", want_logits=True)
    rel = lambda a, ref, lg: np.abs(a.reshape(-1).astype(np.float64) - ref.reshape(-1)) / SO.mol_sensitivity(lg)
    d = rel(nll, pins["trained_nll"], lg)
    print(f"{name} trained Tacotron fixture: max |nll - reference| / sensitivity {d.max():.3e} median {np.median(d):.3e} (bound {TRAINED_TOL})")
    assert name == "simt-fp32" and d.max() <= TRAINED_TOL
    model = helpers.make_model(0, "MOL", "cpu")
    sd = helpers.state_numpy(model)
    mel = pins["rand_mel"]
    m_up, aux = O.upsample_network(sd, O.pad_time(mel.T, 2).T, pad=2)
    x = pins["rand_x"]
    nll, name, lg = score_rows(model.to("cuda"), m_up, aux, x[None], n_seg=1, seg_len=x.size, seg_stride=x.size,
                               precision="fp32", engine="simt", want_logits=True)
    d = rel(nll[0], pins["rand_nll"], lg)
    print(f"{name} random-init fixture: max |nll - reference| / sensitivity {d.max():.3e} (bound {RAND_TOL})")
    assert d.max() <= RAND_TOL


def test_quality_on_trained_checkpoint(trained):
    """fp16 / bf16 scoring on both tensor-core engines against SIMT fp32 on the shipped checkpoint, pinned against the
    CPU emulation's logits at each precision through the same loss."""
    g = trained["g"]
    kw = dict(n_seg=4, seg_len=12100, seg_stride=11550)
    ref, _ = score_rows(trained["model"], trained["m_up"], trained["aux"], g["raw"], precision="fp32", engine="simt", **kw)
    w = O.hot_weights(trained["sd"])
    stats = lambda v: (float(np.median(v)), float(v.mean()), float((np.abs(v - ref) > 1.0).mean()))
    print(f"simt-fp32: median {np.median(ref):.4f} mean {ref.mean():.4f}")
    results = []
    for prec in PRECISIONS:
        _, lg = C.generate_segments(w, trained["m_up"], trained["aux"], steps=12100, mode="MOL", x_force=g["raw"].T.copy(),
                                    uniforms=np.full((12100, 44), 0.5, np.float32), want_logits=True, precision=prec, **kw)
        emu = SO.mol_loss(lg.reshape(-1, 30), g["raw"].T.reshape(-1)).reshape(12100, 4).T
        e_med, e_mean, e_moved = stats(emu)
        for engine in ("tcgen05", "stream"):
            nll, name = score_rows(trained["model"], trained["m_up"], trained["aux"], g["raw"], precision=prec, engine=engine, **kw)
            med, mean, moved = stats(nll)
            print(f"{name}: median {med:.4f} mean {mean:.4f} moved>1nat {moved:.5f} | CPU emulation {prec}: median {e_med:.4f} "
                  f"mean {e_mean:.4f} moved>1nat {e_moved:.5f}")
            results.append((name, med, mean, moved, e_med, e_mean, e_moved))
    # The median sits in the body of the distribution (cdf_delta far above 1e-5), where the loss is well conditioned.
    # The mean is carried by the tail samples whose log-scales reach the clamp: there a logit's last bit moves the loss
    # by hundreds of nats (score_oracle.mol_sensitivity), so it is reported, not pinned.
    for name, med, mean, moved, e_med, e_mean, e_moved in results:
        assert abs(med - e_med) <= 0.01, name
        assert moved <= 1.5 * e_moved + 1e-3, name


# ---------------------------------------------------------------------------------------------------------------------
# mel level
# ---------------------------------------------------------------------------------------------------------------------
TS, NS = (30, 45, 25), (8000, 12000, 6875)      # frames and scored samples per utterance (the last: all T * hop rows)


def utterances(head, Ts=TS, ns=NS, seed=0):
    rs = np.random.RandomState(seed)
    mels = [rs.rand(80, T).astype(np.float32) for T in Ts]
    if head == "MOL":
        xs = [np.clip(0.5 * np.sin(np.arange(n) / 13.0 + i) + 0.05 * rs.randn(n), -1, 1).astype(np.float32) for i, n in enumerate(ns)]
    else:
        xs = [(2.0 * rs.randint(0, 512, n) / 511.0 - 1.0).astype(np.float32) for n in ns]
    return mels, xs


def score_many_device(eng, mels, xs):
    dev = torch.device("cuda", 0)
    dm = [torch.as_tensor(m, device=dev) for m in mels]
    dx = [torch.as_tensor(x, device=dev) for x in xs]
    dn = [torch.full((x.size,), float("nan"), device=dev) for x in xs]
    eng.score_many(mels=[m.data_ptr() for m in dm], Ts=[m.shape[1] for m in mels], xs=[x.data_ptr() for x in dx],
                   ns=[x.size for x in xs], nlls=[o.data_ptr() for o in dn], stream=torch.cuda.current_stream(dev).cuda_stream)
    torch.cuda.synchronize(dev)
    eng.check()
    return [o.cpu().numpy() for o in dn]


def score_frames(eng, mel, x):
    """wrnn_score fed wrnn_conditioning_frames' tensors: one fold of the whole stream."""
    dev = torch.device("cuda", 0)
    T, hop = mel.shape[1], eng.hop_length
    d_mel = torch.as_tensor(mel, device=dev)
    mf, af, taps = torch.empty((T + 4, 80), device=dev), torch.empty((T, 128), device=dev), torch.empty((hop, 5), device=dev)
    s = torch.cuda.current_stream(dev).cuda_stream
    eng.conditioning_frames(mel=d_mel.data_ptr(), T=T, mel_frames=mf.data_ptr(), aux_frames=af.data_ptr(), up_taps=taps.data_ptr(), stream=s)
    d_x = torch.as_tensor(x, device=dev)
    nll = torch.full((x.size,), float("nan"), device=dev)
    eng.score(L=T * hop, n_seg=1, seg_len=x.size, seg_stride=x.size, x_force=d_x.data_ptr(), nll=nll.data_ptr(),
              mel_frames=mf.data_ptr(), aux_frames=af.data_ptr(), up_taps=taps.data_ptr(), hop=hop, stream=s)
    torch.cuda.synchronize(dev)
    eng.check()
    return nll.cpu().numpy()


MEL_LEVEL = [("MOL", "tcgen05", "fp16"), ("RAW", "tcgen05", "bf16"), ("MOL", "simt", "fp32"), ("RAW", "simt", "fp16"),
             ("MOL", "stream", "fp16")]


@pytest.mark.parametrize("head,engine,precision", MEL_LEVEL, ids=[f"{h}-{e}-{p}" for h, e, p in MEL_LEVEL])
def test_score_many(st, head, engine, precision):
    m = st.model(head)[0]
    eng = cabi.Engine(m.hot_state(), n_classes=m.n_classes, mode=head, precision=precision, engine=engine)
    try:
        eng.attach_upsampler(m.state_dict())
        mels, xs = utterances(head)
        batch = score_many_device(eng, mels, xs)
        name = eng.name
        for i in range(len(mels)):
            assert np.isfinite(batch[i]).all()
            alone = score_many_device(eng, [mels[i]], [xs[i]])[0]
            assert np.array_equal(alone, batch[i]), (name, i, "alone")
            if engine != "simt":                         # the SIMT engine takes per-sample rows only
                assert np.array_equal(score_frames(eng, mels[i], xs[i]), batch[i]), (name, i, "conditioning_frames")
        host = eng.score_many_host(mels, xs)
        assert all(np.array_equal(a, b) for a, b in zip(host, batch)), (name, "host")
        perm = [2, 0, 1]
        pb = score_many_device(eng, [mels[i] for i in perm], [xs[i] for i in perm])
        assert all(np.array_equal(pb[k], batch[i]) for k, i in enumerate(perm)), (name, "permuted")
        print(f"score_many {head} [{name}]: {len(mels)} utterances bit-identical alone / frames / host / permuted; "
              f"mean nll {[float(b.mean()) for b in batch]}")
    finally:
        eng.close()


MANY = [("MOL", "fp16"), ("RAW", "bf16")]


@pytest.mark.parametrize("head,precision", MANY, ids=[f"{h}-{p}" for h, p in MANY])
def test_score_many_70_recordings_on_the_persistent_engine(st, head, precision):
    """70 recordings on a fixed persistent handle: a 64-fold launch, then 6 folds.  The batch equals the host entry, and
    the recordings at both ends of each launch equal themselves scored alone."""
    m = st.model(head)[0]
    eng = cabi.Engine(m.hot_state(), n_classes=m.n_classes, mode=head, precision=precision, engine="tcgen05")
    try:
        eng.attach_upsampler(m.state_dict())
        Ts = [2 + i % 4 for i in range(70)]
        mels, xs = utterances(head, Ts, [T * 275 - 13 * (i % 7) for i, T in enumerate(Ts)], seed=3)
        n0 = eng.launch_count
        batch = score_many_device(eng, mels, xs)
        launches = eng.launch_count - n0
        assert eng.name == f"tcgen05-{precision}" and launches == 2, (eng.name, launches)
        assert all(np.isfinite(b).all() for b in batch)
        host = eng.score_many_host(mels, xs)
        assert all(np.array_equal(a, b) for a, b in zip(host, batch)), (eng.name, "host")
        for i in (0, 63, 64, 69):
            alone = score_many_device(eng, [mels[i]], [xs[i]])[0]
            assert np.array_equal(alone, batch[i]), (eng.name, i, "alone")
        print(f"score_many {head} [{eng.name}]: 70 recordings in {launches} launches, bit-identical to the host entry and "
              f"recordings 0, 63, 64, 69 alone")
    finally:
        eng.close()


def test_score_many_auto_routes_many_utterances_to_stream(st):
    m = st.model("MOL")[0]
    n = 257
    rs = np.random.RandomState(5)
    mels = [rs.rand(80, 3).astype(np.float32) for _ in range(n)]
    xs = [np.clip(0.3 * rs.randn(600), -1, 1).astype(np.float32) for _ in range(n)]
    engines = [cabi.Engine(m.hot_state(), n_classes=30, mode="MOL", precision="fp16", engine=e) for e in ("auto", "stream")]
    try:
        for e in engines:
            e.attach_upsampler(m.state_dict())
        auto = engines[0].score_many_host(mels, xs)
        assert engines[0].name.startswith("tcgen05-stream")
        fixed = engines[1].score_many_host(mels, xs)
        assert all(np.array_equal(a, b) for a, b in zip(auto, fixed))
        with pytest.raises(cabi.EngineError, match="upsampler"):
            bare = cabi.Engine(m.hot_state(), n_classes=30, mode="MOL", precision="fp16", engine="tcgen05")
            try:
                bare.score_many_host(mels[:1], xs[:1])
            finally:
                bare.close()
    finally:
        for e in engines:
            e.close()
