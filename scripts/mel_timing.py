"""Throughput of wrnn_melspectrogram_many on an LJSpeech-sized batch: about 13,100 utterances of about 6.6 s at 22050 Hz
(lengths and samples generated on the device from a seed), analysed in one call with the reference's hparams, timed
with CUDA events after a warm-up call of the same batch.  Prints one JSON line: frames/s, the kernel time and the lower
bound on it -- the larger of the FP64 operations over the data-sheet FP64 rate (34 TFLOP/s, H100 SXM, vector) and the
bytes that must move (each sample read once, each mel value written once) over 3.35 TB/s -- with the card's name and
power limit read in the same run.

    python scripts/mel_timing.py [--utts 13100] [--seconds 6.6] [--repeats 3] [--out results/mel_timing.json]"""
import argparse
import json
import math
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

FP64_RATE, HBM_RATE = 34e12, 3.35e12


def frame_flops(n_fft, band_weights):
    """FP64 operations of one frame as the kernel computes it: the window (n_fft multiplies), the radix-2 Stockham
    stages on n_fft / 2 points (10 per butterfly), the unpacking of the n_fft / 2 + 1 bins (about 12 each) and the band
    sums (2 per filterbank weight)."""
    H = n_fft // 2
    return n_fft + 10 * (H // 2) * int(math.log2(H)) + 12 * (H + 1) + 2 * band_weights


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    name, power = (q.stdout.strip().splitlines()[0].split(", ") + ["?"])[:2] if q.returncode == 0 else ("?", "?")
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=13100)
    ap.add_argument("--seconds", type=float, default=6.6)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import numpy as np
    import torch

    from wavernn_b200 import cabi
    assert torch.cuda.is_available(), "mel_timing.py measures on a GPU"
    dev = torch.device("cuda", 0)
    an = cabi.MelAnalysis()
    sr, hop, nm = an.cfg.sample_rate, an.cfg.hop_length, an.cfg.n_mels
    rs = np.random.RandomState(0)
    ns = np.clip(rs.normal(a.seconds, 2.0, a.utts), 1.0, 10.1) * sr
    ns = ns.astype(np.int64)
    g = torch.Generator(device=dev)
    g.manual_seed(0)
    y = (0.1 * torch.randn(int(ns.sum()), generator=g, device=dev)).clamp_(-1, 1)
    Ts = 1 + ns // hop
    mel = torch.empty(int(nm * Ts.sum()), device=dev)
    y0 = np.concatenate([[0], np.cumsum(ns)])
    m0 = np.concatenate([[0], np.cumsum(nm * Ts)])
    ys = [y.data_ptr() + 4 * int(o) for o in y0[:-1]]
    mels = [mel.data_ptr() + 4 * int(o) for o in m0[:-1]]
    s = torch.cuda.current_stream(dev)

    def run():
        an.melspectrogram_many(ys=ys, ns=ns.tolist(), mels=mels, stream=s.cuda_stream)

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
    name, power = card()
    lib = cabi.load()
    import ctypes
    basis = np.zeros((nm, an.cfg.n_fft // 2 + 1))
    lib.wrnn_debug_mel_tables(ctypes.byref(an.cfg), None, basis.ctypes.data, None)
    frames = int(Ts.sum())
    flops = frames * frame_flops(an.cfg.n_fft, int((basis > 0).sum()))
    bytes_ = 4 * int(ns.sum()) + 4 * nm * frames
    t = min(times)
    bound = max(flops / FP64_RATE, bytes_ / HBM_RATE)
    res = dict(metric="mel_frames_per_s", value=frames / t, utterances=a.utts, audio_hours=float(ns.sum() / sr / 3600),
               frames=frames, kernel_s=t, times_s=times, fp64_flop=flops, bytes=bytes_, bound_s=bound,
               bound_by="fp64" if flops / FP64_RATE >= bytes_ / HBM_RATE else "hbm", share_of_bound=bound / t,
               realtime_factor=float(ns.sum() / sr) / t, gpu=name, power_limit=power)
    line = json.dumps(res)
    print(line)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(line + "\n")
    an.close()


if __name__ == "__main__":
    main()
