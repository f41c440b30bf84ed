"""Times scoring (wrnn_score) against generation (wrnn_generate) of the same job on the same handle: microseconds per
step, CUDA events around each call, median of --runs after a warm-up.  Random-init weights (seed 0), random rows,
Philox draws for generation, teacher-forced targets for scoring; steps per fold --steps.

  persistent engine (fixed handle): MoL and RAW at 8, 19 and 64 folds
  stream engine (fixed handle):     MoL at 512 and 4096 folds

Prints one JSON line per measurement, with the card it ran on (name, power limit, maximum SM clock from nvidia-smi).

    python scripts/score_timing.py [--runs 5] [--steps 2000]"""
import argparse
import contextlib
import io
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from wavernn_b200 import WaveRNN, cabi  # noqa: E402

CTOR = dict(rnn_dims=512, fc_dims=512, bits=9, pad=2, upsample_factors=(5, 5, 11), feat_dims=80, compute_dims=128,
            res_out_dims=128, res_blocks=10, hop_length=275, sample_rate=22050)
CASES = [("tcgen05", "MOL", 8), ("tcgen05", "MOL", 19), ("tcgen05", "MOL", 64), ("tcgen05", "RAW", 8), ("tcgen05", "RAW", 19),
         ("tcgen05", "RAW", 64), ("stream", "MOL", 512), ("stream", "MOL", 4096)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return dict(gpu=q[0], power_limit_w=float(q[1]), max_sm_clock_mhz=int(q[2]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--steps", type=int, default=2000)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    info = card()
    models = {}
    for engine, head, n in CASES:
        if head not in models:
            torch.manual_seed(0)
            with contextlib.redirect_stdout(io.StringIO()):
                models[head] = WaveRNN(mode=head, **CTOR).to(dev)
        m = models[head]
        eng = cabi.Engine(m.hot_state(), n_classes=m.n_classes, mode=head, precision="fp16", engine=engine)
        S = a.steps
        g = torch.Generator(device=dev).manual_seed(1)
        L = n * S
        m_up = torch.rand((L, 80), device=dev, generator=g)
        aux = torch.randn((L, 128), device=dev, generator=g)
        x = (torch.randint(0, 512, (S, n), device=dev, generator=g).float() * (2.0 / 511.0) - 1.0).contiguous()
        out = torch.empty((n, S), device=dev)
        nll = torch.empty((S, n), device=dev)
        s = torch.cuda.current_stream(dev).cuda_stream
        kw = dict(mels_up=m_up.data_ptr(), aux=aux.data_ptr(), L=L, n_seg=n, seg_len=S, seg_stride=S, stream=s)
        calls = {"generate": lambda: eng.generate(out=out.data_ptr(), philox_seed=7, **kw),
                 "score": lambda: eng.score(x_force=x.data_ptr(), nll=nll.data_ptr(), **kw)}
        res = {}
        for what, call in calls.items():
            call()
            torch.cuda.synchronize(dev)
            eng.check()
            times = []
            for _ in range(a.runs):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                call()
                e1.record()
                torch.cuda.synchronize(dev)
                eng.check()
                times.append(e0.elapsed_time(e1) * 1e3 / S)
            res[what] = statistics.median(times)
        print(json.dumps(dict(engine=eng.name, head=head, folds=n, steps=S, us_per_step_generate=round(res["generate"], 3),
                              us_per_step_score=round(res["score"], 3), score_over_generate=round(res["score"] / res["generate"], 4),
                              **info)), flush=True)
        eng.close()


if __name__ == "__main__":
    main()
