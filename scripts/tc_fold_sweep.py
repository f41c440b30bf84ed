"""Times MoL jobs on the persistent (tcgen05) engine across fold counts: in-kernel Philox draws, frame-rate conditioning
(the library forms the rows from mel frames, MelResNet frames and the 5-tap table), every one of a fold's 12,100 steps
(target 11,000, overlap 550).  Each point is run 3 times after a warm-up and timed with CUDA events; a separate pass
with WRNN_TC_PROF set then reads CTA 0's cycle counters (fold thread: phases A-E; issuing warp: poll, gather wait, chain
issue, all per step).  Prints one JSON line per fold count with microseconds per step, the cycle counters and the card
it ran on (name, power limit, maximum SM clock from nvidia-smi).

The default fold counts cover one, two and three 8-fold row groups of the small tile (8, 16, 24), the headline job's
19 folds, and the BIG tile at its first (25) and last (64) fold count.

    python scripts/tc_fold_sweep.py [--folds 8 16 19 24 25 64] [--runs 3] [--precision fp16]"""
import argparse
import contextlib
import io
import json
import os
import re
import subprocess
import sys
import tempfile
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from wavernn_b200 import WaveRNN, cabi  # noqa: E402

TARGET, OVERLAP, HOP = 11_000, 550, 275
PROF_KEYS = ("A", "B", "C", "D", "E", "poll", "gather", "issue")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return dict(gpu=q[0], power_limit_w=float(q[1]), max_sm_clock_mhz=int(q[2]))


@contextlib.contextmanager
def stderr_to(path):
    """Points file descriptor 2 (where the library prints its counters) at `path` for the duration."""
    sys.stderr.flush()
    saved = os.dup(2)
    with open(path, "w") as f:
        os.dup2(f.fileno(), 2)
    try:
        yield
    finally:
        sys.stderr.flush()
        os.dup2(saved, 2)
        os.close(saved)


def parse_prof(text):
    """The last `[wrnn_tc prof]` line: cycles per step of CTA 0, keyed by PROF_KEYS."""
    lines = [ln for ln in text.splitlines() if ln.startswith("[wrnn_tc prof]")]
    assert lines, "the library printed no cycle counters"
    vals = [int(v) for v in re.findall(r"=(-?\d+)", lines[-1].split("|", 1)[1])]
    assert len(vals) == len(PROF_KEYS), lines[-1]
    return dict(zip(PROF_KEYS, vals))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--folds", type=int, nargs="+", default=[8, 16, 19, 24, 25, 64])
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=TARGET + 2 * OVERLAP)
    ap.add_argument("--precision", default="fp16", choices=["fp16", "bf16"])
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    info = card()
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        model = WaveRNN(rnn_dims=512, fc_dims=512, bits=9, pad=2, upsample_factors=(5, 5, 11), feat_dims=80, compute_dims=128,
                        res_out_dims=128, res_blocks=10, hop_length=HOP, sample_rate=22050, mode="MOL").to(dev).eval()
    stride, seg_len = TARGET + OVERLAP, TARGET + 2 * OVERLAP
    eng = cabi.Engine(model.hot_state(), n_classes=30, mode="MOL", precision=a.precision, engine="tcgen05", device=0)
    os.environ.pop("WRNN_TC_PROF", None)
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

        def launch(steps):
            eng.generate(mels_up=0, aux=0, L=T * HOP, n_seg=n, seg_len=seg_len, seg_stride=stride, out=out.data_ptr(),
                         steps=steps, philox_seed=7, mel_frames=mel_fr.data_ptr(), aux_frames=aux_fr.data_ptr(),
                         up_taps=taps.data_ptr(), hop=HOP, stream=torch.cuda.current_stream(dev).cuda_stream)

        def finish():
            torch.cuda.synchronize(dev)
            eng.check()

        launch(200)                                      # warm-up: first launch, L2
        finish()
        times = []
        for _ in range(a.runs):
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            launch(a.steps)
            t1.record()
            finish()
            times.append(t0.elapsed_time(t1) * 1e3)
        # the counter pass: one more run, its cycle counters printed by the library's check()
        with tempfile.TemporaryDirectory() as tmp:
            log = Path(tmp) / "prof.txt"
            os.environ["WRNN_TC_PROF"] = "1"
            try:
                with stderr_to(log):
                    launch(a.steps)
                    finish()
            finally:
                os.environ.pop("WRNN_TC_PROF", None)
            prof = parse_prof(log.read_text())
        best = min(times)
        print(json.dumps(dict(folds=n, engine=eng.name, steps=a.steps, runs=a.runs, us_per_step=round(best / a.steps, 3),
                              us_per_step_all=[round(t / a.steps, 3) for t in times],
                              samples_per_s=round(n * a.steps / (best * 1e-6)),
                              cta0_cycles_per_step=prof, **info)), flush=True)
        del mel, mp, mel_fr, aux_fr, out
    eng.close()


if __name__ == "__main__":
    main()
