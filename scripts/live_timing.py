"""Times live unbatched vocoding (wrnn_vocode_live_start / _poll) against wrnn_vocode_host(batched=0) on the same mel and
the same handle: the shipped LJSpeech checkpoint, fp16, persistent engine, a mel of --frames frames (the Tacotron
fixture mels laid end to end), one fold of frames * 275 steps.

  first audio: host clock from just before wrnn_vocode_live_start to the first poll with n_ready > 0 (polls of 100 us)
  us per step: CUDA events around the whole job, divided by its steps.  Live: recorded before _start and right after it
               (so after the kernel in stream order); vocode_host: around the call (it also copies the mel in, runs the
               device epilogue and copies the waveform out, ~1 ms of a ~1.6 s job).  Alternating, --runs of each.
  real-time factor: (1 / 22,050 Hz) / live us per step.

Checks that each live waveform is bit-identical to vocode_host's.  Prints one JSON line with the card it ran on (name,
power limit, maximum SM clock from nvidia-smi).

    python scripts/live_timing.py [--runs 3] [--frames 800]"""
import argparse
import contextlib
import ctypes
import io
import json
import statistics
import subprocess
import sys
import time
import zipfile
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from wavernn_b200 import WaveRNN, cabi  # noqa: E402

CTOR = dict(rnn_dims=512, fc_dims=512, bits=9, pad=2, upsample_factors=(5, 5, 11), feat_dims=80, compute_dims=128,
            res_out_dims=128, res_blocks=10, hop_length=275, sample_rate=22050)
GOLDEN = ROOT / "tests" / "golden"


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return dict(gpu=q[0], power_limit_w=float(q[1]), max_sm_clock_mhz=int(q[2]))


def checkpoint():
    with zipfile.ZipFile(GOLDEN / "pretrained" / "ljspeech.wavernn.mol.800k.zip") as z:
        return torch.load(io.BytesIO(z.read("latest_weights.pyt")), map_location="cpu")


def long_mel(frames):
    g = np.load(GOLDEN / "tacotron_mels.npz")
    mels = [g[f"mel_{i:02d}"].astype(np.float32) / np.float32(65535.0) for i in range(16)]
    mel = np.concatenate(mels * (frames // sum(m.shape[1] for m in mels) + 1), axis=1)[:, :frames]
    return np.ascontiguousarray(mel)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--frames", type=int, default=800)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    info = card()
    with contextlib.redirect_stdout(io.StringIO()):
        m = WaveRNN(mode="MOL", **CTOR)
    m.load_state_dict(checkpoint())
    eng = cabi.Engine(m.hot_state(), n_classes=m.n_classes, mode="MOL", precision="fp16", engine="tcgen05")
    eng.attach_upsampler(m.state_dict())
    lib = eng.lib
    mel = long_mel(a.frames)
    T, steps = mel.shape[1], mel.shape[1] * CTOR["hop_length"]
    wave_len = (T - 1) * CTOR["hop_length"]

    def host():
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        wav = eng.vocode_host(mel, batched=False, philox_seed=11)
        e1.record()
        torch.cuda.synchronize(dev)
        return e0.elapsed_time(e1) * 1e3 / steps, wav

    def live():
        wav = np.full(wave_len, np.nan)
        job = cabi.WrnnVocodeJob(mel.ctypes.data, T, 0, 0, 0, 0, 11, wav.ctypes.data)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n, first, polls = ctypes.c_int64(0), None, 0
        e0.record()
        t0 = time.perf_counter()
        cabi._check(lib, lib.wrnn_vocode_live_start(eng._h, ctypes.byref(job), None))
        e1.record()
        while True:
            rc = lib.wrnn_vocode_live_poll(eng._h, 100, ctypes.byref(n))
            polls += 1
            if first is None and n.value > 0:
                first = (time.perf_counter() - t0, n.value)
            if rc != 1:
                cabi._check(lib, rc)
                break
        torch.cuda.synchronize(dev)
        return e0.elapsed_time(e1) * 1e3 / steps, wav, first, polls

    host()                                               # warm-up: modules, scratch, pinned buffer
    live()
    t_host, t_live, firsts = [], [], []
    for _ in range(a.runs):
        th, want = host()
        tl, got, first, polls = live()
        assert np.array_equal(got.view(np.int64), want.view(np.int64)), "live waveform differs from vocode_host's"
        t_host.append(th)
        t_live.append(tl)
        firsts.append(first)
    us_live, us_host = statistics.median(t_live), statistics.median(t_host)
    print(json.dumps(dict(engine=eng.name, frames=T, steps=steps, runs=a.runs,
                          us_per_step_live=[round(x, 3) for x in t_live], us_per_step_vocode_host=[round(x, 3) for x in t_host],
                          live_over_host=round(us_live / us_host, 4),
                          first_audio_ms=[round(f[0] * 1e3, 3) for f in firsts], first_audio_samples=[f[1] for f in firsts],
                          polls_last_run=polls, real_time_factor=round(1e6 / CTOR["sample_rate"] / us_live, 2),
                          bit_identical=True, **info)), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
