"""Times the C ABI's mel-to-waveform path against the PyTorch one on the same card.

  conditioning: wrnn_conditioning_frames (padded mel + MelResNet on the device, fp32 FFMA) against the eval-mode
                `upsample.resnet` on CUDA (cuDNN, torch's default TF32 setting), at cfg2's 800 and cfg5's 172,034 frames;
                CUDA events, median of --runs after a warm-up.
  end to end:   Engine.vocode_host (host mel in, host float64 wav out) against WaveRNN.generate(gen_rng='philox') on
                cfg2 (10 s mel, MoL) and cfg3 (same mel, 9-bit RAW head with mu-law); target 11,000, overlap 550, random-init
                weights (seed 0), torch.rand mel (seed 0); wall clock, median of --runs after a warm-up.

Prints one JSON line per measurement, with the card it ran on (name, power limit, maximum SM clock from nvidia-smi).

    python scripts/c_vocode_timing.py [--runs 5]"""
import argparse
import contextlib
import io
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from wavernn_b200 import WaveRNN, cabi  # noqa: E402

CTOR = dict(rnn_dims=512, fc_dims=512, bits=9, pad=2, upsample_factors=(5, 5, 11), feat_dims=80, compute_dims=128,
            res_out_dims=128, res_blocks=10, hop_length=275, sample_rate=22050)
TARGET, OVERLAP = 11_000, 550


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return dict(gpu=q[0], power_limit_w=float(q[1]), max_sm_clock_mhz=int(q[2]))


def model(mode, dev):
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        m = WaveRNN(mode=mode, **CTOR)
    m.gen_verbose = False
    m.gen_rng = "philox"
    return m.to(dev)


def engine(m, dev):
    eng = cabi.Engine(m.hot_state(), n_classes=m.n_classes, mode=m.mode, device=dev.index or 0)
    eng.attach_upsampler(m.state_dict())
    return eng


def cuda_ms(fn, runs):
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(runs):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return statistics.median(out), out


def wall_s(fn, runs):
    fn()
    out = []
    for _ in range(runs):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append(time.perf_counter() - t0)
    return statistics.median(out), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    hw = card()
    m = model("MOL", dev)
    eng = engine(m, dev)
    stream = lambda: torch.cuda.current_stream(dev).cuda_stream
    for T in (800, 172_034):
        torch.manual_seed(0)
        mel = torch.rand(1, 80, T, device=dev)
        mel_frames = torch.empty(T + 4, 80, device=dev)
        aux_frames = torch.empty(T, 128, device=dev)
        lib_ms, lib_all = cuda_ms(lambda: eng.conditioning_frames(mel=mel.data_ptr(), T=T, mel_frames=mel_frames.data_ptr(),
                                                                  aux_frames=aux_frames.data_ptr(), stream=stream()), args.runs)
        padded = torch.nn.functional.pad(mel, (2, 2))
        with torch.no_grad():
            torch_ms, torch_all = cuda_ms(lambda: m.upsample.resnet(padded), args.runs)
        print(json.dumps(dict(measure="conditioning", frames=T, library_ms=round(lib_ms, 4), torch_resnet_ms=round(torch_ms, 4),
                              library_runs_ms=[round(x, 4) for x in lib_all], torch_runs_ms=[round(x, 4) for x in torch_all],
                              torch_cudnn_allow_tf32=torch.backends.cudnn.allow_tf32, **hw)), flush=True)
    for cfg, mode in (("cfg2", "MOL"), ("cfg3", "RAW")):
        mm = model(mode, dev)
        e = engine(mm, dev)
        torch.manual_seed(0)
        mel = torch.rand(1, 80, 800)
        mu_law = mode == "RAW"
        host = mel[0].numpy()
        lib_s, lib_all = wall_s(lambda: e.vocode_host(host, target=TARGET, overlap=OVERLAP, mu_law=mu_law), args.runs)
        gen_s, gen_all = wall_s(lambda: mm.generate(mel, None, True, TARGET, OVERLAP, mu_law), args.runs)
        n = 799 * 275
        print(json.dumps(dict(measure="end_to_end", workload=cfg, mode=mode, frames=800, samples=n, vocode_host_s=round(lib_s, 4),
                              generate_philox_s=round(gen_s, 4), vocode_host_runs_s=[round(x, 4) for x in lib_all],
                              generate_runs_s=[round(x, 4) for x in gen_all], engine=e.name, **hw)), flush=True)
        e.close()


if __name__ == "__main__":
    main()
