"""Throughput of wrnn_resample_many to the reference's 22,050 Hz: one batch of --utts recordings of about 6.6 s at each
of 44.1, 48 and 16 kHz (lengths and content generated on the device from a seed), each batch one call, timed with CUDA
events after a warm-up call of the same batch (which also uploads the filter table).  Prints one JSON line: output
samples/s and audio seconds per second for each batch, and the lower bound on the call's time from its FP64
operations (the tap count times 7 per tap when downsampling, 5 when upsampling) over the data-sheet FP64 rate
(34 TFLOP/s, H100 SXM, vector), with the card's name and power limit read in the same run.

    python scripts/resample_timing.py [--utts 2000] [--seconds 6.6] [--repeats 3] [--out results/resample.json]"""
import argparse
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "scripts"))

from mel_timing import FP64_RATE, card  # noqa: E402

NUM_TABLE, NWIN = 2 ** 16, 64 * 2 ** 16 + 1   # wrnn_resample.cu


def mean_taps(sr_in, sr_out, n_probe=20000):
    """Taps per output sample away from the edges, counted as the kernel counts them over n_probe outputs."""
    import numpy as np
    ratio = sr_out / sr_in
    scale = min(1.0, ratio)
    step = int(scale * NUM_TABLE)
    tr = np.arange(10 ** 6, 10 ** 6 + n_probe) * (1.0 / ratio)
    frac = scale * (tr - tr.astype(np.int64))
    taps = (NWIN - (frac * NUM_TABLE).astype(np.int64)) // step + (NWIN - ((scale - frac) * NUM_TABLE).astype(np.int64)) // step
    return float(taps.mean())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=2000)
    ap.add_argument("--seconds", type=float, default=6.6)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import numpy as np
    import torch

    from wavernn_b200 import cabi
    assert torch.cuda.is_available(), "resample_timing.py measures on a GPU"
    dev = torch.device("cuda", 0)
    an = cabi.MelAnalysis()
    sr_out = an.cfg.sample_rate
    s = torch.cuda.current_stream(dev)

    def measure(sr, seed):
        rs = np.random.RandomState(seed)
        ns = (np.clip(rs.normal(a.seconds, 2.0, a.utts), 1.0, 10.1) * sr).astype(np.int64)
        outs = [an.resample_length(int(n), sr) for n in ns]
        g = torch.Generator(device=dev)
        g.manual_seed(seed)
        x = torch.rand(int(ns.sum()), generator=g, device=dev) * 2 - 1
        y = torch.empty(sum(outs), device=dev)
        x0, y0 = np.concatenate([[0], np.cumsum(ns)]), np.concatenate([[0], np.cumsum(outs)])
        xs = [x.data_ptr() + 4 * int(o) for o in x0[:-1]]
        ys = [y.data_ptr() + 4 * int(o) for o in y0[:-1]]

        def run():
            an.resample_many(xs=xs, ns=[int(n) for n in ns], rates=[sr] * a.utts, ys=ys, stream=s.cuda_stream)

        run()                                               # warm-up: module load, table upload, the same batch
        torch.cuda.synchronize(dev)
        times = []
        for _ in range(a.repeats):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(s)
            run()
            e1.record(s)
            torch.cuda.synchronize(dev)
            times.append(e0.elapsed_time(e1) / 1e3)
        t, n_out = min(times), int(y0[-1])
        taps = mean_taps(sr, sr_out)
        flops = n_out * taps * (7 if sr > sr_out else 5)
        del x, y
        return dict(sample_rate=sr, utterances=a.utts, input_samples=int(x0[-1]), output_samples=n_out,
                    audio_s=n_out / sr_out, call_s=t, times_s=times, output_samples_per_s=n_out / t,
                    realtime_factor=n_out / sr_out / t, taps_per_output=taps, fp64_flop=flops,
                    fp64_bound_s=flops / FP64_RATE, share_of_fp64_bound=flops / FP64_RATE / t)

    sets = [measure(sr, i) for i, sr in enumerate((44100, 48000, 16000))]
    name, power = card()
    res = dict(metric="resample_output_samples_per_s", value=sets[0]["output_samples_per_s"], batches=sets, gpu=name,
               power_limit=power)
    line = json.dumps(res)
    print(line)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(line + "\n")
    an.close()


if __name__ == "__main__":
    main()
