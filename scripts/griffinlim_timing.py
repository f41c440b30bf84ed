"""Throughput of wrnn_griffinlim_many at 32 iterations (the reference's reconstruct_waveform default) on two batches:
the 16 Tacotron mels of tests/golden/tacotron_mels.npz, and an LJSpeech-sized batch of --utts mels of about 6.6 s
(lengths and content generated on the device from a seed).  Each batch is one call with the reference's hparams, timed
with CUDA events after a warm-up call of the same batch.  Prints one JSON line: frames/s and audio seconds per second
for each batch, and the lower bound on the call's time from its FP64 operations over the data-sheet FP64 rate
(34 TFLOP/s, H100 SXM, vector), with the card's name and power limit read in the same run.

    python scripts/griffinlim_timing.py [--utts 512] [--seconds 6.6] [--iters 32] [--repeats 3] [--out results/gl.json]"""
import argparse
import ctypes
import json
import math
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "scripts"))
sys.path.insert(0, str(ROOT / "tests"))

from mel_timing import FP64_RATE, card  # noqa: E402

NNLS_ITERS = 100   # wrnn_mel.cu


def fft_flops(n_fft):
    """One radix-2 Stockham transform of n_fft / 2 complex points: 10 operations per butterfly."""
    H = n_fft // 2
    return 10 * (H // 2) * int(math.log2(H))


def frame_flops(n_fft, hop, band_weights, n_iter):
    """FP64 operations of one frame: the solve (2 per filterbank weight for A y, about 9 per bin for A^T r and the
    step, per iteration), then per Griffin-Lim iteration the analysis (window, transform, 12 per bin to unpack), the
    inverse transform (about 14 per point to pack, transform, 3 per sample to unpack and window) and the overlap-add
    (3 per overlapping sample); the final inverse transform and overlap-add once more."""
    nb = n_fft // 2 + 1
    solve = NNLS_ITERS * (2 * band_weights + 9 * nb)
    analysis = n_fft + fft_flops(n_fft) + 12 * nb
    inverse = 14 * (n_fft // 2) + fft_flops(n_fft) + 3 * n_fft + 3 * n_fft
    return solve + n_iter * (analysis + inverse) + inverse


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=512)
    ap.add_argument("--seconds", type=float, default=6.6)
    ap.add_argument("--iters", type=int, default=32)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import numpy as np
    import torch

    import helpers
    from wavernn_b200 import cabi
    assert torch.cuda.is_available(), "griffinlim_timing.py measures on a GPU"
    dev = torch.device("cuda", 0)
    an = cabi.MelAnalysis()
    sr, hop, nm, n_fft = an.cfg.sample_rate, an.cfg.hop_length, an.cfg.n_mels, an.cfg.n_fft
    lib = cabi.load()
    basis = np.zeros((nm, n_fft // 2 + 1))
    lib.wrnn_debug_mel_tables(ctypes.byref(an.cfg), None, basis.ctypes.data, None)
    weights = int((basis > 0).sum())
    s = torch.cuda.current_stream(dev)

    def measure(mel_tensors):
        Ts = [int(m.shape[1]) for m in mel_tensors]
        wav = torch.empty(sum(an.samples(T) for T in Ts), device=dev)
        w0 = np.concatenate([[0], np.cumsum([an.samples(T) for T in Ts])])
        wavs = [wav.data_ptr() + 4 * int(o) for o in w0[:-1]]

        def run():
            an.griffinlim_many(mels=[m.data_ptr() for m in mel_tensors], Ts=Ts, seeds=list(range(len(Ts))), wavs=wavs,
                               n_iter=a.iters, stream=s.cuda_stream)

        run()                                               # warm-up: module load, the same batch
        torch.cuda.synchronize(dev)
        times = []
        for _ in range(a.repeats):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(s)
            run()
            e1.record(s)
            torch.cuda.synchronize(dev)
            times.append(e0.elapsed_time(e1) / 1e3)
        frames, t = sum(Ts), min(times)
        flops = frames * frame_flops(n_fft, hop, weights, a.iters)
        return dict(utterances=len(Ts), frames=frames, audio_s=float(w0[-1] / sr), call_s=t, times_s=times,
                    frames_per_s=frames / t, realtime_factor=float(w0[-1] / sr) / t, fp64_flop=flops,
                    fp64_bound_s=flops / FP64_RATE, share_of_fp64_bound=flops / FP64_RATE / t)

    taco = measure([torch.as_tensor(m, device=dev) for m in helpers.tacotron_mels()])
    rs = np.random.RandomState(0)
    Ts = (np.clip(rs.normal(a.seconds, 2.0, a.utts), 1.0, 10.1) * sr / hop).astype(np.int64) + 1
    g = torch.Generator(device=dev)
    g.manual_seed(0)
    big = torch.rand(int(nm * Ts.sum()), generator=g, device=dev)
    m0 = np.concatenate([[0], np.cumsum(nm * Ts)])
    lj = measure([big[int(m0[i]):int(m0[i + 1])].view(nm, int(Ts[i])) for i in range(a.utts)])
    name, power = card()
    res = dict(metric="griffinlim_frames_per_s", value=lj["frames_per_s"], n_iter=a.iters, tacotron16=taco,
               ljspeech_batch=lj, gpu=name, power_limit=power)
    line = json.dumps(res)
    print(line)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(line + "\n")
    an.close()


if __name__ == "__main__":
    main()
