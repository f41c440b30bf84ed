"""The job matrix that runs every compiled tensor-core kernel (tests/test_gpu_instantiations.py) and every SIMT engine
path (tests/test_gpu_simt.py), the emulation of each job (oracle/contract.py) and the logit tolerances, which the CPU
predicts (tests/test_contract.py).

Every job is teacher-forced with explicit draws and has the edges where the kernels' per-instantiation code differs:
  - seg_stride 271 against a hop of 275: fold windows start at many phases of the hop and cross frame boundaries;
  - steps < seg_len, seg_first != 0;
  - the stream ends half way into the last fold's window, which reads zero rows from there on;
  - fold tables (frame-rate jobs): starts that are not multiples of the stride, windows that end mid-frame and before
    `steps`, one window shorter than 8 rows.
Rows come from frame-rate tensors through the 5-tap table, in float64 (`contract.expand_rows`); the materialised jobs
read those rows rounded to float32.

Every job is made at the reference's hop of 275 (upsample factors (5, 5, 11)) unless given another geometry of
GEOMETRIES, whose taps come from a WaveRNN built with those factors (`geometry_taps`).  The stride stays 271, coprime
with every hop here, so fold windows still start at many phases."""
from __future__ import annotations

import numpy as np

import helpers
from oracle import contract as C
from oracle import philox as P
from test_gpu_sampling import forced_inputs

HOP, STRIDE, STEPS, SEG_LEN, SEG_FIRST = 275, 271, 32, 300, 7
SEED, OFFSET = (3 << 32) | 11, 0x55
PERSISTENT_FOLDS = (24, 25, 73)          # last small tile, first BIG tile, a 64-fold BIG tile then a 9-fold small one
STREAM_FOLDS = {16: 17, 32: 33}          # two tiles of NF folds per CTA, the second one ragged
SMALL_TILE = 24

# Teacher-forced logits of a kernel against contract.generate_segments at the kernel's operand precision.  Each bound is
# at least 4 x the largest float32-vs-float64 accumulation spread of the emulation on these jobs (asserted on the CPU in
# tests/test_contract.py, which prints the spreads: fp16 8.9e-5 MoL / 1.1e-4 RAW, bf16 6.9e-4 / 7.5e-4, fp32 (the SIMT
# engine's strict mode) 1.6e-7 / 1.8e-7), with room for another CPU's float32 summation order; fp16 stays under the
# suite's 1e-3.
LOGIT_TOL = {("fp16", "MOL"): 6e-4, ("fp16", "RAW"): 6e-4, ("bf16", "MOL"): 4e-3, ("bf16", "RAW"): 4e-3,
             ("fp32", "MOL"): 1.2e-6, ("fp32", "RAW"): 1.2e-6}
# fp32 logits against wavernn_oracle.generate_segments (the reference's own operation order, unfolded): at least 4 x
# the largest difference between the fp32 emulation (float32 or float64 sums) and that order on these jobs
# (tests/test_contract.py: 1.8e-7 MoL / 2.1e-7 RAW).
ORACLE_TOL = {"MOL": 1.5e-6, "RAW": 1.5e-6}
# A 16-bit kernel's mean logit error against the emulation at its own precision must be at most 1 / ROUNDING_SEPARATION
# of its mean error against the other 16-bit precision's emulation.  The max-error bounds above cannot tell bf16 from
# fp16 rounding on these jobs; the means can (tests/test_contract.py: the float64-summed emulation, standing in for a
# kernel with another sum order, is 14 x (bf16) and 22 x (fp16) closer to its own precision).
ROUNDING_SEPARATION = 4

# upsampling geometries other than (5, 5, 11) whose impulse response fits the 5-tap table: hop -> upsample factors.
# Hop 1 wraps the phase on every row; at hop <= 8 every 8-row staging group crosses a frame boundary; at 600 a window
# of STEPS rows lies within one or two frames.  200, 256 and 300 are the hops of common 16 / 24 kHz checkpoints.
GEOMETRIES = {1: (1,), 3: (3,), 8: (8,), 9: (3, 3), 200: (5, 5, 8), 256: (4, 8, 8), 300: (5, 6, 10), 600: (600,)}
KERNEL_HOPS = (1, 3, 200, 256, 600)      # the hops besides 275 at which the GPU runs every job (tests/test_gpu_geometries.py)


def geometry_model(hop, mode="MOL", seed=0, **kw):
    """helpers.make_model's network with the upsample factors of GEOMETRIES[hop] (hop 275: helpers.CTOR's)."""
    import contextlib
    import io

    import torch
    from wavernn_b200 import WaveRNN
    factors = helpers.CTOR["upsample_factors"] if hop == HOP else GEOMETRIES[hop]
    torch.manual_seed(seed)
    with contextlib.redirect_stdout(io.StringIO()):
        m = WaveRNN(mode=mode, **dict(helpers.CTOR, upsample_factors=factors, hop_length=hop, **kw))
    m.gen_verbose = False
    return m


def geometry_taps(hop):
    """(hop, 5) float32 interpolation table of the geometry (WaveRNN.upsample_taps on the CPU)."""
    import torch
    m = geometry_model(hop, rnn_dims=32, fc_dims=32)
    taps = m.upsample_taps(torch.device("cpu")).numpy()
    assert m._taps_exact and taps.shape == (hop, 5)
    return taps


def geometry(n, hop=HOP):
    """(L, T): the stream ends half way into the last fold's window; T frames cover it."""
    L = (SEG_FIRST + n - 1) * STRIDE + STEPS // 2
    return L, L // hop + 1


def frames(n, seed, hop=HOP):
    """Padded mel frames (T + 4, 80) and aux frames (T + 4, 128), float32."""
    _, T = geometry(n, hop)
    rs = np.random.RandomState(seed)
    return rs.rand(T + 4, 80).astype(np.float32), rs.randn(T + 4, 128).astype(np.float32)


def fold_tables(n, seed, hop=HOP):
    """fold_row0 / fold_row_end (int64, absolute rows of the stream) for n folds."""
    L, _ = geometry(n, hop)
    rs = np.random.RandomState(seed)
    row0 = rs.randint(0, L - 2 * STEPS, n).astype(np.int64)
    row0[row0 % STRIDE == 0] += 1
    length = rs.randint(STEPS // 2, 2 * STEPS, n)          # about a third end before `steps`
    length[1] = 5                                          # shorter than one 8-row group
    end = np.minimum(row0 + length, L)
    if hop > 1:                                            # (at hop 1 every row starts a frame)
        end[end % hop == 0] -= 1                           # every window ends mid-frame
    return row0, end.astype(np.int64)


def make_job(n, mode, taps, tables=False, hop=HOP):
    """Everything a kernel and the emulation need for one job of n folds at `hop` (taps: that geometry's (hop, 5)
    table).  Strided: `m_up` / `aux` are the job's rows from its first fold on (row SEG_FIRST * STRIDE of the stream), as
    the materialised path indexes them.  Tables: the whole stream, indexed by the absolute fold_row0."""
    L, T = geometry(n, hop)
    seed = 1000 * n + (2 if tables else 0) + (mode == "RAW")
    mel_fr, aux_fr = frames(n, seed, hop)
    row_lo = 0 if tables else SEG_FIRST * STRIDE
    m, a = C.expand_rows(mel_fr, aux_fr, taps, hop, row_lo, L - row_lo)
    job = dict(n=n, mode=mode, tables=tables, hop=hop, L=L, T=T, mel_frames=mel_fr, aux_frames=aux_fr, taps=np.asarray(taps, np.float32),
               row_lo=row_lo, m_up=m.astype(np.float32), aux=a.astype(np.float32), x_force=forced_inputs(n, STEPS, seed + 7),
               fold_row0=None, fold_row_end=None, uniforms=None, expo=None)
    if tables:
        job["fold_row0"], job["fold_row_end"] = fold_tables(n, seed + 3, hop)
    if mode == "MOL":
        job["uniforms"] = P.mol_uniforms(SEED, OFFSET, SEG_FIRST, n, STEPS)
    else:
        job["expo"] = P.raw_expo(SEED, OFFSET, SEG_FIRST, n, STEPS)[0]
    return job


def emulate(w, job, precision, accumulate="f32"):
    """contract.generate_segments on the job: (samples (n, STEPS), logits (STEPS, n, classes))."""
    return C.generate_segments(w, job["m_up"], job["aux"], n_seg=job["n"], seg_len=SEG_LEN, seg_stride=STRIDE, steps=STEPS,
                               mode=job["mode"], uniforms=job["uniforms"], expo=job["expo"], x_force=job["x_force"],
                               fold_row0=job["fold_row0"], fold_row_end=job["fold_row_end"], want_logits=True,
                               precision=precision, accumulate=accumulate)


def oracle_rows(job):
    """The job's rows re-laid out as STEPS-row windows, one per fold, zero past each window's end: the rows fold f reads
    at step t are rows f * STEPS + t, so that wavernn_oracle.generate_segments (which has no fold tables) runs every job
    at seg_stride = STEPS."""
    n, t = job["n"], np.arange(STEPS)
    if job["tables"]:
        row, end = job["fold_row0"][:, None] + t, job["fold_row_end"][:, None]
    else:
        row, end = np.arange(n)[:, None] * STRIDE + t, job["m_up"].shape[0]
    ok = (row < end).reshape(-1, 1)
    r = np.where(ok[:, 0], row.reshape(-1), 0)
    return np.where(ok, job["m_up"][r], 0).astype(np.float32), np.where(ok, job["aux"][r], 0).astype(np.float32)


def emulate_oracle(w, job):
    """wavernn_oracle.generate_segments on the job (its rows by oracle_rows): (samples, logits) as emulate returns them."""
    from oracle import wavernn_oracle as O
    m, a = oracle_rows(job)
    return O.generate_segments(w, m, a, n_seg=job["n"], seg_len=STEPS, seg_stride=STEPS, steps=STEPS, mode=job["mode"],
                               uniforms=job["uniforms"], expo=job["expo"], x_force=job["x_force"], want_logits=True)


def all_jobs():
    """(n, tables) of every job the GPU matrix emulates."""
    return [(n, t) for n in PERSISTENT_FOLDS + tuple(STREAM_FOLDS.values()) for t in (False, True)]


def slice_folds(job, a, b):
    """The draws, teacher inputs and fold tables of folds [a, b) of a job, as a job of b - a folds starting at fold a
    (seg_first + a) would take them."""
    n = job["n"]
    out = {"x_force": np.ascontiguousarray(job["x_force"][:, a:b])}
    u = job["uniforms"]
    out["uniforms"] = None if u is None else np.ascontiguousarray(np.concatenate([u[:, 10 * a:10 * b], u[:, 10 * n + a:10 * n + b]], 1))
    out["expo"] = None if job["expo"] is None else np.ascontiguousarray(job["expo"][:, a:b])
    out["fold_row0"] = None if job["fold_row0"] is None else job["fold_row0"][a:b].copy()
    out["fold_row_end"] = None if job["fold_row_end"] is None else job["fold_row_end"][a:b].copy()
    return out
