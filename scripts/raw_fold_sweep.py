"""Times 9-bit RAW jobs on the persistent (tcgen05) and stream engines across fold counts: in-kernel Philox draws,
frame-rate conditioning (the library forms the rows from mel frames, MelResNet frames and the 5-tap table), every one
of a fold's 12,100 steps (target 11,000, overlap 550).  The two engines alternate within one process, each point is
run 3 times after a warm-up and timed with CUDA events.  Prints one JSON line per (folds, engine) with microseconds
per step, samples per second and the card it ran on (name, power limit, maximum SM clock from nvidia-smi).

    python scripts/raw_fold_sweep.py [--folds 64 256 512 1024 4096] [--runs 3]"""
import argparse
import contextlib
import io
import json
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from wavernn_b200 import WaveRNN, cabi  # noqa: E402

TARGET, OVERLAP, HOP = 11_000, 550, 275


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return dict(gpu=q[0], power_limit_w=float(q[1]), max_sm_clock_mhz=int(q[2]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--folds", type=int, nargs="+", default=[64, 256, 512, 1024, 4096])
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=TARGET + 2 * OVERLAP)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    info = card()
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        model = WaveRNN(rnn_dims=512, fc_dims=512, bits=9, pad=2, upsample_factors=(5, 5, 11), feat_dims=80, compute_dims=128,
                        res_out_dims=128, res_blocks=10, hop_length=HOP, sample_rate=22050, mode="RAW").to(dev).eval()
    stride, seg_len = TARGET + OVERLAP, TARGET + 2 * OVERLAP
    engines = {e: cabi.Engine(model.hot_state(), n_classes=512, mode="RAW", precision="fp16", engine=e, device=0)
               for e in ("tcgen05", "stream")}
    for n in a.folds:
        L = (n - 1) * stride + seg_len
        T = -(-L // HOP)
        mel = torch.rand(1, 80, T, device=dev)
        with torch.no_grad():
            mp = torch.nn.functional.pad(mel, (2, 2))
            mel_fr = mp[0].transpose(0, 1).contiguous()
            aux_fr = model.upsample.resnet(mp)[0].transpose(0, 1).contiguous()
            taps = model.upsample_taps(dev)
        out = torch.empty((n, a.steps), device=dev)

        def launch(eng, steps):
            eng.generate(mels_up=0, aux=0, L=T * HOP, n_seg=n, seg_len=seg_len, seg_stride=stride, out=out.data_ptr(),
                         steps=steps, philox_seed=7, mel_frames=mel_fr.data_ptr(), aux_frames=aux_fr.data_ptr(),
                         up_taps=taps.data_ptr(), hop=HOP, stream=torch.cuda.current_stream(dev).cuda_stream)

        for eng in engines.values():                     # warm-up: first launch, cluster occupancy, L2
            launch(eng, 200)
            torch.cuda.synchronize(dev)
            eng.check()
        times = {e: [] for e in engines}
        for _ in range(a.runs):
            for e, eng in engines.items():
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0.record()
                launch(eng, a.steps)
                t1.record()
                torch.cuda.synchronize(dev)
                eng.check()
                times[e].append(t0.elapsed_time(t1) * 1e3)
        for e, eng in engines.items():
            best = min(times[e])
            print(json.dumps(dict(folds=n, engine=eng.name, steps=a.steps, runs=a.runs, us_per_step=round(best / a.steps, 3),
                                  us_per_step_all=[round(t / a.steps, 3) for t in times[e]],
                                  samples_per_s=round(n * a.steps / (best * 1e-6)), **info)), flush=True)
        del mel, mp, mel_fr, aux_fr, out
    for eng in engines.values():
        eng.close()


if __name__ == "__main__":
    main()
