"""Host side of the drop-in: a `WaveRNN` with the reference's constructor, state_dict
layout and `generate(mels, save_path, batched, target, overlap, mu_law)` signature
(reference models/fatchord_version.py:92-264), whose sample loop is the persistent
sm_90a kernel behind include/wavernn_b200.h instead of ~43 PyTorch launches per
sample.

What stays in PyTorch (run once per call, as the reference does): the
UpsampleNetwork (:64-89).  What stays in numpy float64 on the host: mu-law expansion,
cross-fade/unfold, the fade-out and the wav write (:243-260).  Everything between
`self.upsample(...)` (:186) and `torch.stack(output)` (:243) is the CUDA engine; there
is no CPU fallback.

RNG contract.  `gen_rng='torch'` (default) reproduces the reference's consumption of
torch's default CPU generator: the two throw-away nn.GRUCell constructions of
:178-179, then per step a (1,B,10) and a (1,B) uniform_(1e-5, 1-1e-5) draw
(utils/distribution.py:106,118) -- drawn here in one call (the CPU stream is
split-invariant) and handed to the kernel, so that under the same torch.manual_seed
the output tracks the reference's CPU output within the tolerance stated in
DESIGN.md.  `gen_rng='philox'` draws inside the kernel (counter-based, keyed by
global fold and step, independent of the rank count).
"""
from __future__ import annotations

import os
import time
from pathlib import Path
from typing import Sequence, Union

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import cabi
from .display import progbar, stream
from .dsp import decode_mu_law, save_wav
from .sharding import FoldGeometry, fold_geometry, gather_segments, shard_folds, unbatched_geometry

LOG_SCALE_MIN = float(np.log(1e-14))


# --------------------------------------------------------------------------------------
# Conditioning network (torch; module / parameter names are the checkpoint wire format)
# --------------------------------------------------------------------------------------
class ResBlock(nn.Module):
    def __init__(self, dims):
        super().__init__()
        self.conv1 = nn.Conv1d(dims, dims, kernel_size=1, bias=False)
        self.conv2 = nn.Conv1d(dims, dims, kernel_size=1, bias=False)
        self.batch_norm1 = nn.BatchNorm1d(dims)
        self.batch_norm2 = nn.BatchNorm1d(dims)

    def forward(self, x):
        y = F.relu(self.batch_norm1(self.conv1(x)))
        return self.batch_norm2(self.conv2(y)) + x


class MelResNet(nn.Module):
    def __init__(self, res_blocks, in_dims, compute_dims, res_out_dims, pad):
        super().__init__()
        self.conv_in = nn.Conv1d(in_dims, compute_dims, kernel_size=2 * pad + 1, bias=False)
        self.batch_norm = nn.BatchNorm1d(compute_dims)
        self.layers = nn.ModuleList([ResBlock(compute_dims) for _ in range(res_blocks)])
        self.conv_out = nn.Conv1d(compute_dims, res_out_dims, kernel_size=1)

    def forward(self, x):
        x = F.relu(self.batch_norm(self.conv_in(x)))
        for block in self.layers:
            x = block(x)
        return self.conv_out(x)


class Stretch2d(nn.Module):
    """Nearest-neighbour repeat of the last two axes (reference :51-61)."""

    def __init__(self, x_scale, y_scale):
        super().__init__()
        self.x_scale, self.y_scale = x_scale, y_scale

    def forward(self, x):
        if self.y_scale != 1:
            x = x.repeat_interleave(self.y_scale, dim=2)
        return x.repeat_interleave(self.x_scale, dim=3)


class UpsampleNetwork(nn.Module):
    def __init__(self, feat_dims, upsample_scales, compute_dims, res_blocks, res_out_dims, pad):
        super().__init__()
        total_scale = int(np.prod(upsample_scales))
        self.total_scale = total_scale
        self.indent = pad * total_scale
        self.resnet = MelResNet(res_blocks, feat_dims, compute_dims, res_out_dims, pad)
        self.resnet_stretch = Stretch2d(total_scale, 1)
        self.up_layers = nn.ModuleList()
        for scale in upsample_scales:          # ModuleList indices 1,3,5 hold the convs (checkpoint keys)
            conv = nn.Conv2d(1, 1, kernel_size=(1, 2 * scale + 1), padding=(0, scale), bias=False)
            conv.weight.data.fill_(1. / (2 * scale + 1))
            self.up_layers.append(Stretch2d(scale, 1))
            self.up_layers.append(conv)

    def stretch_mel(self, m):
        """(b, feat, t) -> (b, feat, t*total_scale), un-cropped."""
        m = m.unsqueeze(1)
        for layer in self.up_layers:
            m = layer(m)
        return m.squeeze(1)

    def forward(self, m):
        aux = self.resnet(m).repeat_interleave(self.total_scale, dim=2)
        m = self.stretch_mel(m)[:, :, self.indent:-self.indent]
        return m.transpose(1, 2), aux.transpose(1, 2)


# --------------------------------------------------------------------------------------
class WaveRNN(nn.Module):
    def __init__(self, rnn_dims, fc_dims, bits, pad, upsample_factors, feat_dims, compute_dims, res_out_dims,
                 res_blocks, hop_length, sample_rate, mode='RAW'):
        super().__init__()
        self.mode = mode
        self.pad = pad
        if mode == 'RAW':
            self.n_classes = 2 ** bits
        elif mode == 'MOL':
            self.n_classes = 30
        else:
            # the reference builds this error without raising it (:103-104); generate() raises it (:239)
            raise RuntimeError("Unknown model mode value - ", mode)
        self._to_flatten = []
        self.rnn_dims = rnn_dims
        self.fc_dims = fc_dims
        self.feat_dims = feat_dims
        self.aux_dims = res_out_dims // 4
        self.hop_length = hop_length
        self.sample_rate = sample_rate

        self.upsample = UpsampleNetwork(feat_dims, upsample_factors, compute_dims, res_blocks, res_out_dims, pad)
        self.I = nn.Linear(feat_dims + self.aux_dims + 1, rnn_dims)
        self.rnn1 = nn.GRU(rnn_dims, rnn_dims, batch_first=True)
        self.rnn2 = nn.GRU(rnn_dims + self.aux_dims, rnn_dims, batch_first=True)
        self._to_flatten += [self.rnn1, self.rnn2]
        self.fc1 = nn.Linear(rnn_dims + self.aux_dims, fc_dims)
        self.fc2 = nn.Linear(fc_dims + self.aux_dims, fc_dims)
        self.fc3 = nn.Linear(fc_dims, self.n_classes)
        self.register_buffer('step', torch.zeros(1, dtype=torch.long))
        self.num_params()
        self._flatten_parameters()

        # ---- knobs of the CUDA engine (not part of the reference surface) ----
        self.gen_rng = 'torch'          # 'torch' (reference-compatible CPU draws) | 'philox' (in-kernel)
        self.gen_precision = 'fp16'     # 'fp16' | 'bf16' tensor-core operands | 'fp32' strict SIMT mode
        self.gen_engine = 'auto'        # 'auto' | 'simt' | 'tcgen05' (weights stationary, lowest latency) | 'stream' (many folds)
        self.gen_philox_seed = 0
        self.gen_native_rng = True      # replay torch's CPU generator natively (self-checked; False = torch operators)
        self.gen_max_draw_bytes = 16 << 30   # bound on the host tensor of reference-compatible RAW draws (see _reference_draws)
        self.gen_stream_draws = True    # MoL parity mode: replay + upload the draws in step chunks WHILE the kernel runs
        self.gen_draw_chunk = 1024      # steps per chunk
        self._copy_stream = None
        self._draw_buf = None
        self.gen_upsample_chunk = 2048  # mel frames per UpsampleNetwork call (bounds HBM intermediates)
        self.gen_epilogue = 'device'      # 'device': wrnn_epilogue (xfade / overlap-add / fade-out in one pass) | 'host': numpy
        self.gen_conditioning = 'kernel'  # 'kernel': frame-rate tensors go to the library, which forms the rows (tcgen05 engine)
        #                                   'torch' : materialise UpsampleNetwork's (T*hop, 208) output like the reference
        self.gen_cond_mode = 0            # cabi.COND_AUTO | COND_EXPAND (HBM-rate pre-pass per tile) | COND_IN_KERNEL
        self.gen_verbose = True
        self.gen_stats = {}             # filled by generate(): timings, engine name, ...
        self._engine = None
        self._engine_key = None

    # ------------------------------------------------------------------ training forward (torch)
    def forward(self, x, mels):
        """Teacher-forced forward (reference :131-167); plain PyTorch, not the hot path."""
        device = next(self.parameters()).device
        self._flatten_parameters()
        self.step += 1
        bsize = x.size(0)
        h1 = torch.zeros(1, bsize, self.rnn_dims, device=device)
        h2 = torch.zeros(1, bsize, self.rnn_dims, device=device)
        mels, aux = self.upsample(mels)
        d = self.aux_dims
        a1, a2, a3, a4 = (aux[:, :, d * i:d * (i + 1)] for i in range(4))
        x = self.I(torch.cat([x.unsqueeze(-1), mels, a1], dim=2))
        res = x
        x, _ = self.rnn1(x, h1)
        x = x + res
        res = x
        x, _ = self.rnn2(torch.cat([x, a2], dim=2), h2)
        x = x + res
        x = F.relu(self.fc1(torch.cat([x, a3], dim=2)))
        x = F.relu(self.fc2(torch.cat([x, a4], dim=2)))
        return self.fc3(x)

    # ------------------------------------------------------------------ engine plumbing
    def hot_state(self) -> dict:
        """The 16 tensors the kernel consumes, keyed as in the checkpoint."""
        sd = {k: v for k, v in self.named_parameters() if not k.startswith('upsample.')}
        return {k: sd[k] for k in cabi.WEIGHT_KEYS}

    def _get_engine(self, device: torch.device) -> 'cabi.Engine':
        hot = self.hot_state()
        key = (str(device), self.gen_precision, self.gen_engine, self.mode, self.n_classes,
               tuple((t.data_ptr(), t._version) for t in hot.values()))
        if self._engine is None or key != self._engine_key:
            if self._engine is not None:
                self._engine.close()
            self._engine = cabi.Engine(hot, rnn_dims=self.rnn_dims, fc_dims=self.fc_dims,
                                       feat_dims=self.feat_dims, aux_dims=self.aux_dims,
                                       n_classes=self.n_classes, mode=self.mode, precision=self.gen_precision,
                                       engine=self.gen_engine, device=device.index or 0)
            self._engine_key = key
        return self._engine

    def _require_cuda(self) -> torch.device:
        device = next(self.parameters()).device
        if device.type != 'cuda':
            raise RuntimeError(
                "wavernn_b200: WaveRNN.generate() runs only on a CUDA (sm_90a) device -- move the model with "
                ".to('cuda'). There is deliberately no CPU fallback.")
        return device

    # ------------------------------------------------------------------ conditioning
    def conditioning(self, mels_padded: torch.Tensor, frame_lo: int, frame_hi: int):
        """Upsampled conditioning rows for OUTPUT frames [frame_lo, frame_hi) -- i.e. samples
        [frame_lo*hop, frame_hi*hop) of what `self.upsample(mels_padded)` (:186) returns --
        computed from a slice of the padded mel with a halo, in chunks of
        `gen_upsample_chunk` frames so the x275 intermediates stay small.
        mels_padded: (1, feat, T + 2*pad).  Returns (rows, feat), (rows, 4*aux) fp32."""
        up, pad, hop = self.upsample, self.pad, self.hop_length
        Tp = mels_padded.size(-1)
        halo = 1
        outs_m, outs_a = [], []
        chunk = max(int(self.gen_upsample_chunk), 8)
        for lo in range(frame_lo, frame_hi, chunk):
            hi = min(lo + chunk, frame_hi)
            lo_p = max(0, lo - halo)
            hi_p = min(Tp, hi + 2 * pad + halo)
            piece = mels_padded[:, :, lo_p:hi_p]
            aux = up.resnet(piece)[:, :, lo - lo_p: hi - lo_p]
            aux = aux.repeat_interleave(up.total_scale, dim=2)
            m = up.stretch_mel(piece)[:, :, (lo + pad - lo_p) * hop:(hi + pad - lo_p) * hop]
            outs_m.append(m[0].transpose(0, 1))
            outs_a.append(aux[0].transpose(0, 1))
        m = torch.cat(outs_m, dim=0) if len(outs_m) > 1 else outs_m[0]
        a = torch.cat(outs_a, dim=0) if len(outs_a) > 1 else outs_a[0]
        return m.contiguous().float(), a.contiguous().float()

    def upsample_taps(self, device) -> torch.Tensor:
        """(hop, 5) fp32: composed impulse response of UpsampleNetwork's three stretch+conv stages (reference
        :73-80) per output phase -- mel_up[n] = sum_d taps[n % hop][d] * mel_padded[n // hop + d].  Obtained by
        pushing a unit impulse through the module's own layers (exact for every sample that survives the
        `indent` crop, :88; checked in tests/test_dropin_api.py).  Cached per weight version."""
        up = self.upsample
        key = (str(device),) + tuple((l.weight.data_ptr(), l.weight._version) for l in up.up_layers if hasattr(l, 'weight'))
        if getattr(self, '_taps_key', None) != key:
            hop, n_fr, c = up.total_scale, 9, 4
            x = torch.zeros(1, 1, n_fr, device=device)
            x[0, 0, c] = 1.0
            with torch.no_grad():
                y = up.stretch_mel(x)[0, 0]                                   # impulse at frame c
            n = torch.arange(n_fr * hop, device=device)
            d = c - n // hop + 2
            keep = (d >= 0) & (d < 5)
            taps = torch.zeros(hop, 5, device=device)
            taps[(n % hop)[keep], d[keep]] = y[keep]
            # the 5-tap form is exact only if the whole impulse response falls inside the table (it does for the
            # reference's (5, 5, 11); a first factor of 1 widens the support beyond +-2 frames)
            self._taps_exact = bool((y[~keep] == 0).all().item())
            self._taps, self._taps_key = taps.contiguous(), key
        return self._taps

    def _kernel_conditioning_ok(self) -> bool:
        """Frame-rate conditioning (rows formed by the library from 5 taps per phase) is served when the engine is the
        tcgen05 one AND the module's geometry is the one the tap table encodes: pad == 2 (the kernels read mel frames
        n//hop .. n//hop + 4 of the (T + 2*pad)-row tensor, i.e. a centre offset of pad = 2) and an interpolation
        cascade whose impulse response fits 5 frames.  Any other `pad` / `upsample_factors` (the reference accepts
        them, fatchord_version.py:64-89) takes the materialised torch path, like the reference."""
        if not (self.gen_conditioning == 'kernel' and self.gen_precision != 'fp32'
                and self.gen_engine in ('auto', 'tcgen05', 'stream') and (self.mode == 'MOL' or self.n_classes == 512)):
            return False
        if self.pad != 2 or self.upsample.total_scale != self.hop_length:
            return False
        self.upsample_taps(next(self.parameters()).device)
        return bool(self._taps_exact)

    # ------------------------------------------------------------------ randomness
    def _reference_draws(self, geo: FoldGeometry, steps: int, reuse_buffer: bool = False, shard=None):
        """Consumes torch's default CPU generator exactly as the reference's generate() does: two nn.GRUCell
        constructions (:178-179, one uniform per parameter element, discarded) and then the loop's draws.
        With `gen_native_rng` the generator is replayed natively (cabi.torch_rng_uniform: the discarded part is skipped,
        the used part written straight into a pinned staging buffer) -- same numbers, same final generator state,
        ~10x less host time; it is self-checked against torch once per process."""
        B = geo.n_seg
        native = bool(self.gen_native_rng) and cabi.is_built() and cabi.torch_rng_replay_ok()
        if native:
            skip = sum(3 * g.hidden_size * (g.input_size + g.hidden_size + 2) for g in (self.rnn1, self.rnn2))
            if self.mode == 'MOL':
                # `shard`: only this rank's folds' columns of the (steps, 11*B) matrix are converted and kept --
                # the result is the (steps, 11*n_local) block the kernel consumes, not the whole matrix
                cols = None
                n_keep = n = steps * 11 * B
                if shard is not None and shard.n_seg < B:
                    f0, nl = shard.seg_first, shard.n_seg
                    cols = ((10 * f0, 10 * (f0 + nl)), (10 * B + f0, 10 * B + f0 + nl))
                    n_keep = steps * 11 * nl
                buf = None
                if torch.cuda.is_available():
                    if reuse_buffer:        # one job at a time: the caller synchronises before the next call
                        if self._draw_buf is None or self._draw_buf.numel() < n_keep:
                            self._draw_buf = torch.empty(n_keep, dtype=torch.float32, pin_memory=True)
                        buf = self._draw_buf
                    else:
                        buf = torch.empty(n_keep, dtype=torch.float32, pin_memory=True)
                u = cabi.torch_rng_uniform(skip, n, 1e-5, 1.0 - 1e-5, out=buf, row_len=11 * B, cols=cols)
                return u[:n_keep].view(steps, n_keep // steps), None
            cabi.torch_rng_uniform(skip, 0, 0.0, 1.0)
        else:
            nn.GRUCell(self.rnn1.input_size, self.rnn1.hidden_size)     # :178 get_gru_cell(self.rnn1)
            nn.GRUCell(self.rnn2.input_size, self.rnn2.hidden_size)     # :179
        if self.mode == 'MOL':
            u = torch.empty(steps, 11 * B).uniform_(1e-5, 1.0 - 1e-5)   # distribution.py:106,118
            return u, None
        # RAW: Categorical.sample() -> torch.multinomial -> one exponential_() of shape (B, n_classes) per step
        # (:233-235).  Only this rank's folds are kept (the whole (B, n_classes) row is still drawn: the stream is
        # the reference's).  512 draws per fold-step is what parity with the reference costs: 25 MB per fold of
        # 12,100 steps -- long RAW jobs should use gen_rng='philox' (in-kernel draws, no host tensor at all).
        f0, nl = (shard.seg_first, shard.n_seg) if shard is not None else (0, B)
        need = steps * nl * self.n_classes * 4
        if need > self.gen_max_draw_bytes:
            raise RuntimeError(f"wavernn_b200: gen_rng='torch' on the RAW head needs {need / 2**30:.1f} GiB of Exp(1) draws for "
                               f"{nl} folds x {steps} steps; set model.gen_rng = 'philox' (or raise model.gen_max_draw_bytes)")
        e = torch.empty(steps, nl, self.n_classes, pin_memory=torch.cuda.is_available())
        row = torch.empty(B, self.n_classes)
        for t in range(steps):
            row.exponential_()
            e[t] = row[f0:f0 + nl]
        return None, e

    def _can_stream_draws(self, steps: int, x_force, draws) -> bool:
        """MoL parity draws can be replayed and uploaded while the kernel runs (wrnn_job::uniforms_ready) when they come
        from the native replay and a tensor-core engine consumes them."""
        # (needs the upload stream to run UNDER the kernel: not when launches are serialised -- CUDA_LAUNCH_BLOCKING=1, or a
        #  kernel profiler such as ncu, for which WRNN_STREAM_DRAWS=0 selects the resident matrix; the kernel would wait for
        #  rows that cannot arrive and end with WRNN_E_WATCHDOG)
        if os.environ.get('CUDA_LAUNCH_BLOCKING', '0') == '1' or os.environ.get('WRNN_STREAM_DRAWS', '1') == '0':
            return False
        return (bool(self.gen_stream_draws) and self.gen_rng == 'torch' and draws is None and x_force is None and self.mode == 'MOL'
                and self.gen_precision != 'fp32' and self.gen_engine != 'simt' and steps > 2 * int(self.gen_draw_chunk)
                and bool(self.gen_native_rng) and cabi.is_built() and cabi.torch_rng_replay_ok())

    @staticmethod
    def _draw_chunk_bounds(steps: int, chunk: int, n_folds: int):
        """Step boundaries of the streamed draw chunks.  The first chunk sits on the critical path (it is replayed before
        the launch): ~128 k draws however many folds the job has, then doubling up to `chunk` steps (the replay is ~16x
        faster than the kernel consumes rows, so every chunk lands long before its first row is read)."""
        first = max(8, min(chunk, (1 << 17) // (11 * n_folds)))
        bounds, size = [0], first
        while bounds[-1] < steps:
            bounds.append(min(steps, bounds[-1] + size))
            size = min(chunk, 2 * size)
        return bounds

    def _streamed_draws(self, geo: FoldGeometry, steps: int, shard, device, launch):
        """The reference's draws (two discarded nn.GRUCell initialisations, then `steps` rows of 11*B uniforms; same
        generator consumption as _reference_draws) replayed natively in chunks of up to `gen_draw_chunk` steps.  Chunk 0 is
        uploaded, then `launch(uniforms_ptr, ready_ptr)` enqueues the kernel, then the remaining chunks are replayed and
        uploaded on a side stream while it runs; after every chunk a 4-byte copy on that stream bumps the device counter
        the kernel checks before it reads a row.  Host replay time (9 ms on an 8-rank job) leaves the critical path."""
        B, f0, nl = geo.n_seg, shard.seg_first, shard.n_seg
        skip = sum(3 * g.hidden_size * (g.input_size + g.hidden_size + 2) for g in (self.rnn1, self.rnn2))
        cols = ((10 * f0, 10 * (f0 + nl)), (10 * B + f0, 10 * B + f0 + nl)) if nl < B else None
        width = 11 * nl
        chunk = int(self.gen_draw_chunk)
        bounds = self._draw_chunk_bounds(steps, chunk, B)
        n_keep = steps * width
        if self._draw_buf is None or self._draw_buf.numel() < n_keep:
            self._draw_buf = torch.empty(n_keep, dtype=torch.float32, pin_memory=True)
        host = self._draw_buf
        marks = torch.tensor(bounds[1:], dtype=torch.int32).pin_memory()
        main = torch.cuda.current_stream(device)
        if self._copy_stream is None or self._copy_stream.device != device:
            self._copy_stream = torch.cuda.Stream(device)
        side = self._copy_stream
        dev = torch.empty(n_keep, dtype=torch.float32, device=device)
        ready = torch.zeros(1, dtype=torch.int32, device=device)
        dev.record_stream(side); ready.record_stream(side)
        side.wait_stream(main)                                   # the counter is zero before the first bump
        for i in range(len(bounds) - 1):
            r0, r1 = bounds[i], bounds[i + 1]
            piece = host[r0 * width:r1 * width]
            cabi.torch_rng_uniform(skip if i == 0 else 0, (r1 - r0) * 11 * B, 1e-5, 1.0 - 1e-5, out=piece, row_len=11 * B, cols=cols)
            with torch.cuda.stream(side):
                dev[r0 * width:r1 * width].copy_(piece, non_blocking=True)
                ready.copy_(marks[i:i + 1], non_blocking=True)
            if i == 0:
                launch(dev.data_ptr(), ready.data_ptr())
        return dev, ready, side

    # ------------------------------------------------------------------ the hot path
    def generate(self, mels, save_path: Union[str, Path, None], batched, target, overlap, mu_law):
        """Same contract as reference :169-264: returns the float64 waveform of length
        (T-1)*hop_length, writes it as a float32 wav to `save_path`, leaves the module in
        train() mode."""
        t_start = time.time()
        self.eval()
        device = self._require_cuda()
        if self.mode not in ('MOL', 'RAW'):
            raise RuntimeError("Unknown model mode value - ", self.mode)
        mu_law = mu_law if self.mode == 'RAW' else False
        dist_on = torch.distributed.is_available() and torch.distributed.is_initialized()
        rank = torch.distributed.get_rank() if dist_on else 0
        world = torch.distributed.get_world_size() if dist_on else 1

        with torch.no_grad():
            mels = torch.as_tensor(mels, device=device).float()
            T = mels.size(-1)
            wave_len = (T - 1) * self.hop_length
            total_len = T * self.hop_length
            mels_padded = F.pad(mels, (self.pad, self.pad))                      # :185
            geo = fold_geometry(total_len, target, overlap) if batched else unbatched_geometry(total_len)
            if not batched:
                world_eff, rank_eff = 1, 0      # a single segment does not shard: replicas only
            else:
                world_eff, rank_eff = world, rank
            shard = shard_folds(geo, rank_eff, world_eff, self.hop_length)

            out_local = self._run_segments(mels_padded, geo, shard, device)
            t_kernel_done = time.time()
            if world_eff > 1:
                out_all = gather_segments(out_local, shard, geo)
            else:
                out_all = out_local
            wav = self._finish(out_all, geo, batched, wave_len, mu_law)          # :243-258
        if save_path is not None and rank == 0:                                  # one writer per job
            save_wav(wav, save_path, self.sample_rate)                           # :260
        self.train()                                                             # :262
        elapsed = time.time() - t_start
        self.gen_stats.update(wall_s=elapsed, loop_wall_s=t_kernel_done - t_start, n_seg=geo.n_seg,
                              seg_len=geo.seg_len, wave_len=wave_len, world=world_eff)
        if self.gen_verbose and rank == 0:
            self.gen_display(geo.seg_len - 1, geo.seg_len, geo.n_seg, t_start)
        return wav

    def _run_segments(self, mels_padded, geo: FoldGeometry, shard, device, *, steps: int = 0,
                      x_force=None, want_logits: bool = False, draws=None):
        """Conditioning for this rank's folds + one persistent-kernel launch.
        Returns the (n_seg_local, S) float32 device tensor of samples (pre-xfade)."""
        S = steps or geo.seg_len
        uniforms = expo = None
        frames = self._kernel_conditioning_ok() and x_force is None and not want_logits and shard.n_seg > 0
        if frames:      # enqueue the frame-rate GPU work first: it overlaps the host-side RNG replay below
            T = mels_padded.size(-1) - 2 * self.pad
            mel_fr = mels_padded[0].transpose(0, 1).contiguous().float()                  # (T + 2 pad, feat)
            aux_fr = self.upsample.resnet(mels_padded)[0].transpose(0, 1).contiguous().float()   # (T, 4*aux)
            taps = self.upsample_taps(device)
        stream_draws = frames and self._can_stream_draws(S, x_force, draws)
        if stream_draws:
            pass                                   # drawn, uploaded and consumed concurrently: see _streamed_draws below
        elif self.gen_rng == 'torch' or draws is not None:
            u_all, e_all = draws if draws is not None else self._reference_draws(geo, S, reuse_buffer=True, shard=shard)
            f0, n = shard.seg_first, shard.n_seg
            B = geo.n_seg
            if u_all is not None:
                u_loc = u_all if u_all.shape[1] == 11 * n else \
                    torch.cat([u_all[:, 10 * f0:10 * (f0 + n)], u_all[:, 10 * B + f0:10 * B + f0 + n]], dim=1)
                uniforms = u_loc.contiguous().to(device, non_blocking=True)
            if e_all is not None:
                e_loc = e_all if e_all.shape[1] == n else e_all[:, f0:f0 + n].contiguous()
                expo = e_loc.to(device, non_blocking=True)
        elif self.gen_rng != 'philox':
            raise ValueError(f"gen_rng must be 'torch' or 'philox', got {self.gen_rng!r}")
        if shard.n_seg == 0:
            return torch.zeros((0, S), dtype=torch.float32, device=device)
        engine = self._get_engine(device)
        out = torch.empty((shard.n_seg, S), dtype=torch.float32, device=device)
        if frames:
            # frame-rate conditioning: the library forms every (T*hop, 208) row itself from the padded mel, the
            # MelResNet frames and the 5-tap interpolation table (an HBM-rate pre-pass per 64-fold tile, or inside the
            # persistent kernel -- cabi.COND_*); torch never materialises anything of size T*hop
            def launch(uni_ptr, ready_ptr):
                engine.generate(mels_up=0, aux=0, L=T * self.hop_length, n_seg=shard.n_seg, seg_len=geo.seg_len,
                                seg_stride=geo.seg_stride, out=out.data_ptr(), seg_first=shard.seg_first, steps=steps,
                                uniforms=uni_ptr, expo=expo.data_ptr() if expo is not None else 0,
                                philox_seed=int(self.gen_philox_seed), mel_frames=mel_fr.data_ptr(),
                                aux_frames=aux_fr.data_ptr(), up_taps=taps.data_ptr(), hop=self.hop_length,
                                cond_mode=int(self.gen_cond_mode), uniforms_ready=ready_ptr,
                                stream=torch.cuda.current_stream(device).cuda_stream)
            if stream_draws:
                keep = self._streamed_draws(geo, S, shard, device, launch)
                keep[2].synchronize()
            else:
                launch(uniforms.data_ptr() if uniforms is not None else 0, 0)
            torch.cuda.current_stream(device).synchronize()
            engine.check()
            self.gen_stats.update(engine=engine.name, grid_ctas=engine.grid_ctas, launches=engine.launch_count,
                                  conditioning='kernel')
            return out
        m_up, aux = self.conditioning(mels_padded, shard.frame_lo, shard.frame_hi)
        off = shard.row_lo - shard.frame_lo * self.hop_length
        n_rows = shard.row_hi - shard.row_lo
        m_up = m_up[off:off + n_rows]
        aux = aux[off:off + n_rows]
        if off:
            m_up, aux = m_up.contiguous(), aux.contiguous()
        logits = (torch.empty((S, shard.n_seg, self.n_classes), dtype=torch.float32, device=device)
                  if want_logits else None)
        xf = None
        if x_force is not None:
            xf = torch.as_tensor(x_force, dtype=torch.float32, device=device).contiguous()
        engine.generate(mels_up=m_up.data_ptr(), aux=aux.data_ptr(), L=n_rows, n_seg=shard.n_seg,
                        seg_len=geo.seg_len, seg_stride=geo.seg_stride, out=out.data_ptr(),
                        seg_first=shard.seg_first, steps=steps,
                        uniforms=uniforms.data_ptr() if uniforms is not None else 0,
                        expo=expo.data_ptr() if expo is not None else 0,
                        philox_seed=int(self.gen_philox_seed), philox_offset=0,
                        x_force=xf.data_ptr() if xf is not None else 0,
                        logits_out=logits.data_ptr() if logits is not None else 0,
                        stream=torch.cuda.current_stream(device).cuda_stream)
        torch.cuda.current_stream(device).synchronize()
        engine.check()
        self.gen_stats.update(engine=engine.name, grid_ctas=engine.grid_ctas, launches=engine.launch_count,
                              conditioning='torch')
        del m_up, aux, uniforms, expo, xf
        return (out, logits) if want_logits else out

    def _finish(self, samples: torch.Tensor, geo: FoldGeometry, batched, wave_len, mu_law) -> np.ndarray:
        """(n_seg, S) fp32 samples -> float64 waveform: on the device (`gen_epilogue='device'`, wrnn_epilogue: one pass,
        bit-identical to the host version by construction) or with the host numpy restatement of :243-258."""
        if (self.gen_epilogue == 'device' and samples.is_cuda and wave_len >= 20 * self.hop_length
                and (not batched or geo.overlap > 0)):
            tabs = self._epilogue_tables(geo, batched, mu_law, samples.device)
            wav = torch.empty(wave_len, dtype=torch.float64, device=samples.device)
            samples = samples.contiguous()
            p = lambda t: 0 if t is None else t.data_ptr()
            cabi.epilogue(samples=samples.data_ptr(), n_seg=samples.shape[0], seg_len=samples.shape[1],
                          seg_stride=geo.seg_stride, overlap=geo.overlap if batched else 0, fade_in=p(tabs['fade_in']),
                          fade_out=p(tabs['fade_out']), mu_table=p(tabs['mu']), n_classes=self.n_classes,
                          tail=p(tabs['tail']), tail_len=20 * self.hop_length, wave_len=wave_len, wav=wav.data_ptr(),
                          stream=torch.cuda.current_stream(samples.device).cuda_stream)
            return wav.cpu().numpy()
        output = samples.cpu().numpy().astype(np.float64)                        # :243-245
        return self._epilogue(output, geo, batched, wave_len, mu_law)

    def _epilogue_tables(self, geo: FoldGeometry, batched, mu_law, device):
        """float64 weight tables of the epilogue, built with the reference's own numpy expressions (:255, :379-391,
        utils/dsp.py:98-103) and cached on the device."""
        key = (geo.overlap if batched else 0, bool(mu_law), self.n_classes, self.hop_length, str(device))
        if getattr(self, '_ep_key', None) != key:
            to = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).to(device)
            fade_in = fade_out = mu = None
            if key[0] > 0:
                silence_len = key[0] // 2
                t = np.linspace(-1, 1, key[0] - silence_len, dtype=np.float64)
                fade_in = np.concatenate([np.zeros(silence_len), np.sqrt(0.5 * (1 + t))])
                fade_out = np.concatenate([np.ones(silence_len), np.sqrt(0.5 * (1 - t))])
            if mu_law:      # the kernel's samples are x_k = 2k/(n-1) - 1 in fp32 (:235): expand exactly those values
                n = self.n_classes
                x32 = np.float32(2) * np.arange(n, dtype=np.float32) / np.float32(n - 1) - np.float32(1)
                mu = decode_mu_law(x32.astype(np.float64), n, False)
            self._ep_tabs = dict(fade_in=to(fade_in), fade_out=to(fade_out), mu=to(mu),
                                 tail=to(np.linspace(1, 0, 20 * self.hop_length)))
            self._ep_key = key
        return self._ep_tabs

    def _epilogue(self, output: np.ndarray, geo: FoldGeometry, batched, wave_len, mu_law) -> np.ndarray:
        """numpy float64 tail of the reference (:247-258)."""
        if mu_law:
            output = decode_mu_law(output, self.n_classes, False)
        output = self.xfade_and_unfold(output, geo.target, geo.overlap) if batched else output[0]
        fade_out = np.linspace(1, 0, 20 * self.hop_length)
        output = output[:wave_len]
        output[-20 * self.hop_length:] *= fade_out
        return output

    def generate_many(self, mels_list: Sequence, save_paths: Sequence, target, overlap, mu_law):
        """Extension (SURVEY 8f-1): vocode several utterances in ONE job.  The reference vocodes sentences one
        at a time (gen_tacotron.py:139-163); here the folds of all utterances share the persistent kernel's
        tiles -- a step costs the same for 1 or 64 folds, so k short utterances cost about one.
        Returns the list of waveforms; each is exactly what `generate(m, path, True, target, overlap, mu_law)`
        returns when the calls are made one after the other under the same torch seed (the per-utterance RNG
        draws are made in that order)."""
        device = self._require_cuda()
        dist_on = torch.distributed.is_available() and torch.distributed.is_initialized()
        rank = torch.distributed.get_rank() if dist_on else 0
        world = torch.distributed.get_world_size() if dist_on else 1
        if self.mode not in ('MOL', 'RAW'):
            raise RuntimeError("Unknown model mode value - ", self.mode)
        if len(mels_list) == 0:
            return []
        mu_law = mu_law if self.mode == 'RAW' else False                        # :174
        t_start = time.time()
        self.eval()
        hop = self.hop_length
        geos, wave_lens, streams_m, streams_a, draws = [], [], [], [], []
        frames = self._kernel_conditioning_ok()          # same conditioning path as generate() -> identical samples
        with torch.no_grad():
            for m in mels_list:
                m = torch.as_tensor(m, device=device).float()
                T = m.size(-1)
                geo = fold_geometry(T * hop, target, overlap)
                geos.append(geo); wave_lens.append((T - 1) * hop)
                mp = F.pad(m, (self.pad, self.pad))
                if frames:       # frame-rate tensors, T + 2*pad rows each so mel and aux share one frame index
                    streams_m.append(mp[0].transpose(0, 1).float())
                    streams_a.append(F.pad(self.upsample.resnet(mp)[0].transpose(0, 1).float(), (0, 0, 0, 2 * self.pad)))
                else:
                    m_up, aux = self.conditioning(mp, 0, T)
                    streams_m.append(m_up); streams_a.append(aux)
                if self.gen_rng == 'torch':
                    draws.append(self._reference_draws(geo, geo.seg_len))        # same order as sequential generate() calls
            S, stride = geos[0].seg_len, geos[0].seg_stride
            B = sum(g.n_seg for g in geos)
            row0, row_end, base = [], [], 0
            for g in geos:                                       # utterance streams laid end to end
                row0 += [base + i * stride for i in range(g.n_seg)]
                row_end += [base + g.total_len] * g.n_seg
                base += g.total_len + (2 * self.pad * hop if frames else 0)
            m_all, a_all = torch.cat(streams_m, 0).contiguous(), torch.cat(streams_a, 0).contiguous()
            if frames:
                # one HBM-rate pre-pass lays the x275 rows of all utterances end to end (same arithmetic as generate()'s
                # per-tile pre-pass -> identical samples); the pad frames between utterances give rows no fold reads
                n_rows = base - 2 * self.pad * hop
                cs = torch.cuda.current_stream(device).cuda_stream
                m_rows = torch.empty((n_rows, m_all.shape[1]), dtype=torch.float32, device=device)
                a_rows = torch.empty((n_rows, a_all.shape[1]), dtype=torch.float32, device=device)
                cabi.expand_conditioning(mel_frames=m_all.data_ptr(), aux_frames=a_all.data_ptr(),
                                         up_taps=self.upsample_taps(device).data_ptr(), hop=hop, row_lo=0, n_rows=n_rows,
                                         mels_up=m_rows.data_ptr(), aux=a_rows.data_ptr(), stream=cs)
                m_all, a_all = m_rows, a_rows
            t_row0 = torch.tensor(row0, dtype=torch.int64, device=device)
            t_end = torch.tensor(row_end, dtype=torch.int64, device=device)
            # the job's folds (all utterances, in order) are sharded over the ranks like generate()'s: contiguous
            # blocks, no data-path collective, one all-gather of the sample blocks
            job = FoldGeometry(base, target, overlap, B, S, stride, base)
            shard = shard_folds(job, rank, world, hop)
            f_lo, n_loc = shard.seg_first, shard.n_seg
            uniforms = expo = None
            if self.gen_rng == 'torch' and self.mode == 'MOL':
                mix = torch.cat([u[:, :10 * g.n_seg] for (u, _), g in zip(draws, geos)], 1)
                logi = torch.cat([u[:, 10 * g.n_seg:] for (u, _), g in zip(draws, geos)], 1)
                uniforms = torch.cat([mix[:, 10 * f_lo:10 * (f_lo + n_loc)], logi[:, f_lo:f_lo + n_loc]], 1) \
                    .contiguous().to(device, non_blocking=True)
            elif self.gen_rng == 'torch':         # RAW: per-utterance Exp(1) streams, folds side by side
                expo = torch.cat([e for _, e in draws], 1)[:, f_lo:f_lo + n_loc].contiguous().to(device, non_blocking=True)
            elif self.gen_rng != 'philox':
                raise ValueError(f"gen_rng must be 'torch' or 'philox', got {self.gen_rng!r}")
            engine = self._get_engine(device)
            out = torch.empty((n_loc, S), dtype=torch.float32, device=device)
            if n_loc:
                cond = dict(mels_up=m_all.data_ptr(), aux=a_all.data_ptr())
                engine.generate(L=m_all.shape[0], n_seg=n_loc, seg_len=S, seg_stride=stride, out=out.data_ptr(), seg_first=f_lo,
                                uniforms=uniforms.data_ptr() if uniforms is not None else 0,
                                expo=expo.data_ptr() if expo is not None else 0,
                                philox_seed=int(self.gen_philox_seed), fold_row0=t_row0[f_lo:].data_ptr(),
                                fold_row_end=t_end[f_lo:].data_ptr(),
                                stream=torch.cuda.current_stream(device).cuda_stream, **cond)
                torch.cuda.current_stream(device).synchronize()
                engine.check()
            if world > 1:
                out = gather_segments(out, shard, job)
        wavs, f0 = [], 0
        for g, wl, path in zip(geos, wave_lens, save_paths):
            wav = self._finish(out[f0:f0 + g.n_seg], g, True, wl, mu_law)
            f0 += g.n_seg
            if path is not None and rank == 0:
                save_wav(wav, path, self.sample_rate)
            wavs.append(wav)
        self.train()
        self.gen_stats.update(wall_s=time.time() - t_start, n_seg=B, seg_len=S, engine=engine.name,
                              launches=engine.launch_count, utterances=len(geos), world=world)
        return wavs

    # ------------------------------------------------------------------ reference helpers kept for callers
    def gen_display(self, i, seq_len, b_size, start):
        gen_rate = (i + 1) / (time.time() - start) * b_size / 1000
        msg = f'| {progbar(i, seq_len)} {i * b_size}/{seq_len * b_size} | Batch Size: {b_size} | ' \
              f'Gen Rate: {gen_rate:.1f}kHz | '
        stream(msg)

    def get_gru_cell(self, gru):
        cell = nn.GRUCell(gru.input_size, gru.hidden_size)
        cell.weight_hh.data = gru.weight_hh_l0.data
        cell.weight_ih.data = gru.weight_ih_l0.data
        cell.bias_hh.data = gru.bias_hh_l0.data
        cell.bias_ih.data = gru.bias_ih_l0.data
        return cell

    def pad_tensor(self, x, pad, side='both'):
        b, t, c = x.size()
        total = t + 2 * pad if side == 'both' else t + pad
        padded = torch.zeros(b, total, c, device=x.device)
        if side in ('before', 'both'):
            padded[:, pad:pad + t, :] = x
        elif side == 'after':
            padded[:, :t, :] = x
        return padded

    def fold_with_overlap(self, x, target, overlap):
        """(1, L, F) -> (num_folds, target + 2*overlap, F); materialised form of the strided
        windows the kernel indexes directly (reference :293-340)."""
        _, total_len, features = x.size()
        geo = fold_geometry(total_len, target, overlap)
        if geo.padded_len != total_len:
            x = self.pad_tensor(x, geo.padded_len - total_len, side='after')
        return x[0].unfold(0, geo.seg_len, geo.seg_stride).permute(0, 2, 1).contiguous()

    def xfade_and_unfold(self, y, target, overlap):
        """Equal-power cross-fade + overlap-add (reference :342-405); mutates y in place like
        the reference does."""
        num_folds, length = y.shape
        target = length - 2 * overlap
        total_len = num_folds * (target + overlap) + overlap
        silence_len = overlap // 2
        fade_len = overlap - silence_len
        t = np.linspace(-1, 1, fade_len, dtype=np.float64)
        fade_in = np.concatenate([np.zeros(silence_len), np.sqrt(0.5 * (1 + t))])
        fade_out = np.concatenate([np.ones(silence_len), np.sqrt(0.5 * (1 - t))])
        y[:, :overlap] *= fade_in
        y[:, -overlap:] *= fade_out
        unfolded = np.zeros(total_len, dtype=np.float64)
        step = target + overlap
        for i in range(num_folds):
            unfolded[i * step:i * step + length] += y[i]
        return unfolded

    def get_step(self):
        return self.step.data.item()

    def log(self, path, msg):
        with open(path, 'a') as f:
            print(msg, file=f)

    def load(self, path: Union[str, Path]):
        device = next(self.parameters()).device
        self.load_state_dict(torch.load(path, map_location=device), strict=False)

    def save(self, path: Union[str, Path]):
        torch.save(self.state_dict(), path)

    def num_params(self, print_out=True):
        n = sum(int(np.prod(p.size())) for p in self.parameters() if p.requires_grad) / 1_000_000
        if print_out:
            print('Trainable Parameters: %.3fM' % n)
        return n

    def _flatten_parameters(self):
        for m in self._to_flatten:
            m.flatten_parameters()
