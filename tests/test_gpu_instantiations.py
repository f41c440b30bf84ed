"""Every compiled tensor-core kernel against the engine-arithmetic emulation (oracle/contract.py), one test per kernel:

  persistent  wrnn_tc_kernel<FMT, FRAMES, RAW, BIG>           fp16 | bf16 x rows | FRAMES x MoL | RAW x small | BIG  (16)
  stream      wrnn_stream_kernel<NF, FMT, FRAMES, CL, RAW>    16 | 32 folds x 1 | 4 CTAs x fp16 | bf16 x rows | FRAMES x MoL | RAW  (32)

FRAMES kernels build the conditioning rows from frame-rate tensors in their staging warps; the others read
materialised rows.  The jobs (tests/kernel_jobs.py) are teacher-forced with explicit draws, their outputs pre-filled
with NaN, and have the edges where these kernels differ: stride 271 against the 275-sample hop, steps < seg_len,
seg_first != 0, a last fold that runs past the end of the stream, fold tables with short and mid-frame windows; persistent jobs of
24, 25 and 73 folds (the last is a 64-fold BIG tile then a 9-fold small tile), stream jobs of NF + 1 folds.

Checks: the kernel that ran (engine name, grid, launches); logits against contract.generate_segments within
kernel_jobs.LOGIT_TOL; samples against the kernel's own logits (RAW: the host argmax; MoL: the SFU error bounds of
test_gpu_sampling); bit-for-bit: FRAMES == rows from the conditioning pre-pass, BIG tile == the same folds as small
tiles, cluster form == one-CTA form.  Run on a GPU: pytest -m gpu -s (one line per kernel)."""
import math
import os

import numpy as np
import pytest
import torch

import helpers
import kernel_jobs as K
from oracle import contract as C
from oracle import wavernn_oracle as O
from test_gpu_sampling import LIBM, LOG_SCALE_MIN, SFU, gumbel_err, kernel_picks, log_err, raw_host_picks
from wavernn_b200 import cabi

pytestmark = pytest.mark.gpu

PRECISIONS, HEADS = ("fp16", "bf16"), ("MOL", "RAW")
PERSISTENT = [(p, h, fr, big) for p in PRECISIONS for h in HEADS for fr in (False, True) for big in (False, True)]
STREAM = [(p, h, fr, nf, cl) for p in PRECISIONS for h in HEADS for fr in (False, True) for nf in (16, 32) for cl in (1, 4)]
MT = 64                                   # folds per persistent launch


class Matrix:
    """Module state: one model per head, the 8 engines, the jobs, their emulations and the runs of the stream engine's
    one-CTA forms (the cluster forms are compared with them)."""

    def __init__(self):
        self.models, self.engines, self.jobs, self.emus, self.runs = {}, {}, {}, {}, {}

    def model(self, head):
        if head not in self.models:
            m = helpers.make_model(0, head)                # taps on the CPU, as tests/test_contract.py predicts with
            w = O.hot_weights(helpers.state_numpy(m))
            taps = m.upsample_taps(torch.device("cpu")).numpy()
            self.models[head] = (m.to("cuda"), w, taps)
        return self.models[head]

    def engine(self, kind, precision, head):
        key = (kind, precision, head)
        if key not in self.engines:
            m = self.model(head)[0]
            self.engines[key] = cabi.Engine(m.hot_state(), n_classes=m.n_classes, mode=head, precision=precision,
                                            engine={"persistent": "tcgen05", "stream": "stream"}[kind], device=0)
        return self.engines[key]

    def job(self, n, head, tables):
        if (n, head, tables) not in self.jobs:
            self.jobs[(n, head, tables)] = K.make_job(n, head, self.model(head)[2], tables)
        return self.jobs[(n, head, tables)]

    def emu(self, precision, n, head, tables):
        key = (precision, n, head, tables)
        if key not in self.emus:
            self.emus[key] = K.emulate(self.model(head)[1], self.job(n, head, tables), precision)
        return self.emus[key]

    def close(self):
        for e in self.engines.values():
            e.close()


@pytest.fixture(scope="module")
def mx():
    m = Matrix()
    yield m
    m.close()


def launch(eng, job, source, *, a=0, b=None, cond_mode=cabi.COND_AUTO, form=None):
    """Folds [a, b) of `job` on `eng`.  source: "rows" (the job's materialised float32 rows), "prepass" (rows formed on
    the device by cabi.expand_conditioning) or "frames" (frame-rate tensors, rows formed by the kernel or, under
    COND_EXPAND, by the persistent engine's own pre-pass).  form: (NF, CL) of the stream engine.
    Returns samples (n, STEPS), logits (STEPS, n, classes), the engine's name, its grid and the launches made."""
    dev = torch.device("cuda", 0)
    b = job["n"] if b is None else b
    n = b - a
    d = K.slice_folds(job, a, b)
    t = lambda x: None if x is None else torch.as_tensor(np.ascontiguousarray(x), device=dev)
    p = lambda x: 0 if x is None else x.data_ptr()
    tables = job["tables"]
    row0, end = t(d["fold_row0"]), t(d["fold_row_end"])
    kw = dict(mels_up=0, aux=0, mel_frames=0, aux_frames=0, up_taps=0, hop=0)
    if source == "frames":
        mel_fr, aux_fr, taps = t(job["mel_frames"]), t(job["aux_frames"]), t(job["taps"])
        kw.update(mel_frames=p(mel_fr), aux_frames=p(aux_fr), up_taps=p(taps), hop=job["hop"])
        L = job["L"]
    else:
        n_rows = job["L"] - job["row_lo"]
        if source == "rows":
            m_up, aux = t(job["m_up"]), t(job["aux"])
        else:
            mel_fr, aux_fr, taps = t(job["mel_frames"]), t(job["aux_frames"]), t(job["taps"])
            m_up = torch.empty((n_rows, 80), device=dev)
            aux = torch.empty((n_rows, 128), device=dev)
            cabi.expand_conditioning(mel_frames=p(mel_fr), aux_frames=p(aux_fr), up_taps=p(taps), hop=job["hop"], row_lo=job["row_lo"],
                                     n_rows=n_rows, mels_up=p(m_up), aux=p(aux), stream=torch.cuda.current_stream(dev).cuda_stream)
        if not tables:                                    # the sub-job's rows start at its first fold
            m_up, aux, n_rows = m_up[a * K.STRIDE:], aux[a * K.STRIDE:], n_rows - a * K.STRIDE
        kw.update(mels_up=p(m_up), aux=p(aux))
        L = n_rows
    nc = 30 if job["mode"] == "MOL" else 512
    out = torch.full((n, K.STEPS), float("nan"), device=dev)
    lg = torch.full((K.STEPS, n, nc), float("nan"), device=dev)
    U, E, X = t(d["uniforms"]), t(d["expo"]), t(d["x_force"])
    saved = {v: os.environ.get(v) for v in ("WRNN_STREAM_NF", "WRNN_STREAM_CL")}
    if form is not None:
        os.environ["WRNN_STREAM_NF"], os.environ["WRNN_STREAM_CL"] = str(form[0]), str(form[1])
    before = eng.launch_count
    try:
        eng.generate(L=L, n_seg=n, seg_len=K.SEG_LEN, seg_stride=K.STRIDE, out=p(out), seg_first=K.SEG_FIRST + a, steps=K.STEPS,
                     uniforms=p(U), expo=p(E), x_force=p(X), logits_out=p(lg), fold_row0=p(row0), fold_row_end=p(end),
                     cond_mode=cond_mode, stream=torch.cuda.current_stream(dev).cuda_stream, **kw)
    finally:
        for v, old in saved.items():
            if old is None:
                os.environ.pop(v, None)
            else:
                os.environ[v] = old
    torch.cuda.synchronize(dev)
    eng.check()
    res, lgs = out.cpu().numpy(), lg.cpu().numpy()
    assert not np.isnan(res).any() and not np.isnan(lgs).any(), "outputs left unwritten"
    return res, lgs, eng.name, eng.grid_ctas, eng.launch_count - before


def check_samples(job, out, lg, a=0, b=None, acc=SFU):
    """Samples against the kernel's own logits and the job's draws, under the error model `acc` of the kernel's
    transcendentals: SFU (the tensor-core kernels' __logf / __expf) or LIBM (the SIMT engine's logf / expf)."""
    d = K.slice_folds(job, a, job["n"] if b is None else b)
    if job["mode"] == "RAW":
        want, margin = raw_host_picks(lg, d["expo"])
        got = kernel_picks(out)
        if acc is SFU:
            bound = 1e-5
        else:
            # the SIMT sampler ranks expf(l - max) / sum / e: per class, log of that is off by at most the rounding of
            # l - max (2^-24 of it), expf's 2 ulp and two divisions' half ulps, < 2^-21 + 2^-24 |l - max|; a pick may
            # differ only where the top two are closer than the sum of two such errors
            bound = 2.0 * (2.0 ** -21 + 2.0 ** -24 * np.ptp(lg.astype(np.float64), axis=-1))
        clear = margin > bound
        assert clear.mean() >= 0.99 and np.array_equal(got[clear], want[clear]), int((got != want)[clear].sum())
        return
    # MoL (utils/distribution.py:106-121 in float64): the sample must be some component's sample within the sampler's
    # tolerance, and that component's Gumbel score within the documented logf error of the best
    S, B = lg.shape[:2]
    U = d["uniforms"]
    mix, ul = U[:, :10 * B].reshape(S, B, 10).astype(np.float64), U[:, 10 * B:].astype(np.float64)
    l = lg.astype(np.float64)
    g = l[..., :10] - np.log(-np.log(mix))
    err = gumbel_err(mix, acc) + 2.0 ** -23 * (np.abs(g) + np.abs(l[..., :10]))
    k = np.argmax(g, axis=-1)[..., None]
    admissible = np.take_along_axis(g, k, -1) - g <= np.take_along_axis(err, k, -1) + err
    mean, s = l[..., 10:20], np.exp(np.maximum(l[..., 20:30], np.float64(LOG_SCALE_MIN)))
    lu = np.log(ul) - np.log1p(-ul)
    dd = s * lu[..., None]
    dev = np.abs(np.clip(mean + dd, -1, 1) - out.T[..., None].astype(np.float64))
    if acc is SFU:     # test_gpu_sampling's SFU tolerance
        consistent = (dev <= 1e-5 * np.maximum(np.abs(mean), np.abs(dd))) | (dev <= s * 2.0 ** -20.41)
    else:
        # logf(u) - logf(1 - u) with 1 ulp per logf, the float rounding of 1 - u (< 2^-24, i.e. < 2^-23 in the log) and
        # of the difference; then expf (2 ulp), the product and the sum: < 2^-21 of |mean| + |term|
        lu_err = log_err(ul, LIBM) + log_err(1 - ul, LIBM) + 2.0 ** -23 + 2.0 ** -24 * np.abs(lu)
        consistent = dev <= s * lu_err[..., None] + 2.0 ** -21 * (np.abs(mean) + np.abs(dd))
    ok = (admissible & consistent).any(-1)
    assert ok.all(), [(int(i), int(j)) for i, j in zip(*np.nonzero(~ok))][:5]


def logit_error(lg, emu_lg, precision, head, what):
    e = float(np.abs(lg.astype(np.float64) - emu_lg).max())
    assert e <= K.LOGIT_TOL[(precision, head)], (what, e)
    return e


# ---------------------------------------------------------------------------------------------------------------------
# persistent engine
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision,head,frames,big", PERSISTENT,
                         ids=[f"tc-{p}-{h}-{'frames' if fr else 'rows'}-{'big' if big else 'small'}" for p, h, fr, big in PERSISTENT])
def test_persistent_kernel(mx, precision, head, frames, big):
    check_persistent_kernel(mx, precision, head, frames, big)


def check_persistent_kernel(mx, precision, head, frames, big, tag=""):
    """The checks of one persistent kernel on mx's jobs; prints one line (prefixed by `tag`)."""
    eng = mx.engine("persistent", precision, head)
    errs = []

    def run(job, source, **kw):
        out, lg, name, grid, launches = launch(eng, job, source, **kw)
        n = kw.get("b", job["n"]) - kw.get("a", 0)
        tiles = math.ceil(n / MT)
        assert name == f"tcgen05-{precision}" and grid == 128
        assert launches == tiles * (2 if kw.get("cond_mode") == cabi.COND_EXPAND else 1), launches
        return out, lg

    for n in ((25, 73) if big else (24,)):
        # the tiles of this job (64 folds each, the last one ragged): one of them runs the kernel under test
        assert any((min(MT, n - f0) > K.SMALL_TILE) == big for f0 in range(0, n, MT))
        for tables in ((False, True) if frames else (False,)):
            job = mx.job(n, head, tables)
            _, emu_lg = mx.emu(precision, n, head, tables)
            if frames:
                cond = cabi.COND_AUTO if tables else cabi.COND_IN_KERNEL
                out, lg = run(job, "frames", cond_mode=cond)
                # the same rows from the conditioning pre-pass, read by the kernel without FRAMES
                if tables:
                    out_p, lg_p = run(job, "prepass")
                else:
                    out_p, lg_p = run(job, "frames", cond_mode=cabi.COND_EXPAND)
                assert np.array_equal(out, out_p) and np.array_equal(lg, lg_p), "FRAMES != pre-pass rows"
            else:
                out, lg = run(job, "rows")
            errs.append(logit_error(lg, emu_lg, precision, head, (n, tables)))
            check_samples(job, out, lg)
            if big and n == 25:
                # the BIG tile's folds as a small tile of 24 and a tile of 1, with their draws and seg_first
                source = "frames" if frames else "rows"
                cond = cabi.COND_IN_KERNEL if frames and not tables else cabi.COND_AUTO
                parts = [run(job, source, a=a, b=b, cond_mode=cond) for a, b in ((0, 24), (24, 25))]
                assert np.array_equal(out, np.concatenate([parts[0][0], parts[1][0]], 0)), "BIG != small (samples)"
                assert np.array_equal(lg, np.concatenate([parts[0][1], parts[1][1]], 1)), "BIG != small (logits)"
    print(f"{tag}persistent {'BIG' if big else 'small'} {'FRAMES' if frames else 'rows'} {precision} {head}: "
          f"max logit error vs emulation {max(errs):.2e} (tolerance {K.LOGIT_TOL[(precision, head)]:.1e})")


# ---------------------------------------------------------------------------------------------------------------------
# stream engine
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision,head,frames,nf,cl", STREAM,
                         ids=[f"stream-{p}-{h}-{'frames' if fr else 'rows'}-{nf}x{cl}" for p, h, fr, nf, cl in STREAM])
def test_stream_kernel(mx, precision, head, frames, nf, cl):
    check_stream_kernel(mx, precision, head, frames, nf, cl)


def check_stream_kernel(mx, precision, head, frames, nf, cl, tag=""):
    """The checks of one stream kernel form on mx's jobs; prints one line (prefixed by `tag`)."""
    eng = mx.engine("stream", precision, head)
    n = K.STREAM_FOLDS[nf]
    errs = []

    def run(job, source, form):
        key = (precision, head, job["tables"], source, form)
        if key not in mx.runs:
            out, lg, name, grid, launches = launch(eng, job, source, form=form)
            assert name == (f"tcgen05-stream-x4-{precision}" if form[1] == 4 else f"tcgen05-stream-{precision}"), name
            assert grid == math.ceil(n / form[0]) * form[1] and launches == 1, (grid, launches)
            mx.runs[key] = (out, lg)
        return mx.runs[key]

    for tables in ((False, True) if frames else (False,)):
        job = mx.job(n, head, tables)
        _, emu_lg = mx.emu(precision, n, head, tables)
        source = "frames" if frames else "rows"
        out, lg = run(job, source, (nf, cl))
        if frames:
            out_p, lg_p = run(job, "prepass", (nf, cl))
            assert np.array_equal(out, out_p) and np.array_equal(lg, lg_p), "FRAMES != pre-pass rows"
        if cl == 4:
            out_1, lg_1 = run(job, source, (nf, 1))
            assert np.array_equal(out, out_1) and np.array_equal(lg, lg_1), "cluster form != one-CTA form"
        errs.append(logit_error(lg, emu_lg, precision, head, tables))
        check_samples(job, out, lg)
    print(f"{tag}stream {nf}x{cl} {'FRAMES' if frames else 'rows'} {precision} {head}: "
          f"max logit error vs emulation {max(errs):.2e} (tolerance {K.LOGIT_TOL[(precision, head)]:.1e})")


# ---------------------------------------------------------------------------------------------------------------------
# the conditioning pre-pass and the heads the engines refuse
# ---------------------------------------------------------------------------------------------------------------------
def test_conditioning_pre_pass_against_the_float64_rows():
    """cabi.expand_conditioning against contract.expand_rows: mel within the error bound of the kernel's 5-fmaf chain
    (2^-21 of the sum of |tap x mel|), aux bit for bit.  Short runs at a non-zero phase, a run long enough for the
    grid-stride loop to go round more than once, and the last row of the stream (mel frames up to T + 3)."""
    model = helpers.make_model(0, "MOL")
    check_pre_pass(model.upsample_taps(torch.device("cpu")).numpy(), 275, 80)


def check_pre_pass(taps, hop, T):
    """The pre-pass on T frames at `hop` with that geometry's taps: runs of 1, 7, 8 and 9 rows from row 3 hop + 101 %
    hop, all rows but the first 57, and the last row."""
    dev = torch.device("cuda", 0)
    rs = np.random.RandomState(9)
    mel_fr, aux_fr = rs.rand(T + 4, 80).astype(np.float32), rs.randn(T, 128).astype(np.float32)
    d_mel, d_aux, d_taps = (torch.as_tensor(x, device=dev) for x in (mel_fr, aux_fr, taps))
    n_sm = torch.cuda.get_device_properties(dev).multi_processor_count
    cases = [(3 * hop + 101 % hop, k) for k in (1, 7, 8, 9)] + [(57, T * hop - 57), (T * hop - 1, 1)]
    assert T * hop - 57 > 2 * 8 * 8 * n_sm                # more than two passes of the capped grid (8 rows per block)
    for row_lo, n_rows in cases:
        m = torch.full((n_rows, 80), float("nan"), device=dev)
        a = torch.full((n_rows, 128), float("nan"), device=dev)
        cabi.expand_conditioning(mel_frames=d_mel.data_ptr(), aux_frames=d_aux.data_ptr(), up_taps=d_taps.data_ptr(), hop=hop,
                                 row_lo=row_lo, n_rows=n_rows, mels_up=m.data_ptr(), aux=a.data_ptr(),
                                 stream=torch.cuda.current_stream(dev).cuda_stream)
        torch.cuda.synchronize(dev)
        m, a = m.cpu().numpy(), a.cpu().numpy()
        want_m, want_a = C.expand_rows(mel_fr, aux_fr, taps, hop, row_lo, n_rows)
        r = np.arange(row_lo, row_lo + n_rows)
        bound = 2.0 ** -21 * sum(np.abs(taps[r % hop, dd].astype(np.float64)[:, None] * mel_fr[r // hop + dd]) for dd in range(5))
        e = np.abs(m - want_m)
        print(f"pre-pass hop {hop} rows [{row_lo}, {row_lo + n_rows}): max mel error {e.max():.2e}, max error / bound {(e / np.maximum(bound, 1e-300)).max():.3f}")
        assert (e <= bound).all() and np.array_equal(a, want_a.astype(np.float32)), (row_lo, n_rows)


@pytest.mark.parametrize("engine", ["auto", "tcgen05", "stream", "simt"])
def test_raw_heads_other_than_9_bits_are_refused(engine):
    """Every engine serves the RAW head at 9 bits (512 classes) only; a 10-bit head is refused with a message, under
    ENGINE_AUTO too (no engine falls back to serving it)."""
    torch.manual_seed(0)
    from wavernn_b200 import WaveRNN
    m = WaveRNN(mode="RAW", **dict(helpers.CTOR, bits=10)).to("cuda")
    assert m.n_classes == 1024
    with pytest.raises(cabi.EngineError, match="512"):
        cabi.Engine(m.hot_state(), n_classes=1024, mode="RAW", precision="fp16", engine=engine, device=0)
