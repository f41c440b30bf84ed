"""Times the C ABI's batch entry against one call per utterance, on the workload of BASELINE configs[3].

  workload: the 16 Tacotron sentences of tests/golden/tacotron_mels.npz, the shipped LJSpeech MoL checkpoint of
            tests/golden/pretrained/, target 11,000, overlap 550 (104 folds as one batch).
  batch:      one Engine.vocode_many_host over the 16 mels (seeds 0..15)
  sequential: 16 Engine.vocode_host calls, one per mel, with the same seeds
  context:    WaveRNN.generate_many(gen_rng='philox') on the same mels
The batch and the sequential calls alternate, on one AUTO handle; wall clock (host mels in, host float64 waveforms out),
median of --runs after a warm-up of each.  Also checks that every batch waveform equals its single call when both are
served by the same engine.

Prints one JSON line per measurement, with the card it ran on (name, power limit, maximum SM clock from nvidia-smi).

    python scripts/c_vocode_many_timing.py [--runs 5]"""
import argparse
import contextlib
import io
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

import helpers  # noqa: E402
from wavernn_b200 import WaveRNN, cabi  # noqa: E402
from wavernn_b200.sharding import fold_geometry  # noqa: E402

TARGET, OVERLAP = 11_000, 550


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return dict(gpu=q[0], power_limit_w=float(q[1]), max_sm_clock_mhz=int(q[2]))


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    hw = card()
    sd = helpers.pretrained_state_dict()
    with contextlib.redirect_stdout(io.StringIO()):
        m = WaveRNN(mode="MOL", **helpers.CTOR)
    m.load_state_dict(sd)
    m = m.to(dev).eval()
    m.gen_verbose = False
    m.gen_rng = "philox"
    mels = helpers.tacotron_mels()
    seeds = list(range(len(mels)))
    folds = sum(fold_geometry(x.shape[1] * 275, TARGET, OVERLAP).n_seg for x in mels)
    eng = cabi.Engine(m.hot_state(), n_classes=m.n_classes, mode=m.mode, device=0)
    eng.attach_upsampler(m.state_dict())

    batch = lambda: eng.vocode_many_host(mels, seeds, target=TARGET, overlap=OVERLAP)
    seq = lambda: [eng.vocode_host(x, target=TARGET, overlap=OVERLAP, philox_seed=s) for x, s in zip(mels, seeds)]
    _, wb = timed(batch)
    batch_engine = eng.name
    _, ws = timed(seq)
    seq_engine = eng.name
    same = all(np.array_equal(a, b) for a, b in zip(wb, ws))
    tb, ts = [], []
    for _ in range(args.runs):
        tb.append(timed(batch)[0])
        ts.append(timed(seq)[0])
    med_b, med_s = statistics.median(tb), statistics.median(ts)
    common = dict(utterances=len(mels), folds=folds, frames=sum(x.shape[1] for x in mels), target=TARGET, overlap=OVERLAP,
                  checkpoint="ljspeech.wavernn.mol.800k", **hw)
    print(json.dumps(dict(measure="vocode_many_host", median_s=round(med_b, 4), runs_s=[round(x, 4) for x in tb],
                          engine=batch_engine, **common)), flush=True)
    print(json.dumps(dict(measure="vocode_host_x16", median_s=round(med_s, 4), runs_s=[round(x, 4) for x in ts],
                          engine=seq_engine, **common)), flush=True)
    print(json.dumps(dict(measure="speedup", sequential_over_batch=round(med_s / med_b, 3),
                          bit_identical_to_single_calls=same, same_engine=batch_engine == seq_engine, **common)), flush=True)

    tm = [torch.from_numpy(x)[None] for x in mels]
    gen = lambda: m.generate_many(tm, [None] * len(tm), TARGET, OVERLAP, False)
    timed(gen)
    tg = [timed(gen)[0] for _ in range(args.runs)]
    print(json.dumps(dict(measure="generate_many_philox", median_s=round(statistics.median(tg), 4),
                          runs_s=[round(x, 4) for x in tg], **common)), flush=True)


if __name__ == "__main__":
    main()
