"""Times live batch vocoding (wrnn_vocode_many_live_start / _poll) against wrnn_vocode_many_host(batched=0) on the same
batch and the same handle: the shipped LJSpeech checkpoint, fp16, persistent engine, n mels of --frames frames each (the
Tacotron fixture mels laid end to end, utterance i starting at fixture mel i), one fold of frames * 275 steps each.

  us per step: CUDA events around the whole job, divided by its steps.  Live: recorded before _start and right after it
               (so after the kernel in stream order); vocode_many_host: around the call (it also copies the mels in, runs
               the device epilogue and copies the waveforms out).  Alternating, --runs of each per batch size.
  first audio: per utterance, host clock from just before _start to the first poll (of 100 us) with n_ready[i] > 0.
  real-time factor of each stream: (1 / 22,050 Hz) / live us per step (every fold makes one sample per step).

At one utterance, wrnn_vocode_live_start (the batch of one on the same route) is timed in the same alternation.  It used
to run one fold on expanded rows; this comparison, made then, retired that route (DESIGN §3.6).  Checks that every live
waveform is bit-identical to vocode_many_host's.  Prints one JSON line per batch size with the card it ran on (name, power limit, maximum SM clock from nvidia-smi).

    python scripts/live_many_timing.py [--runs 3] [--frames 800] [--sizes 1,8,24,25,64]"""
import argparse
import contextlib
import ctypes
import io
import json
import statistics
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "scripts"))

from live_timing import CTOR, GOLDEN, card, checkpoint  # noqa: E402
from wavernn_b200 import WaveRNN, cabi  # noqa: E402


def mels_of(n, frames):
    g = np.load(GOLDEN / "tacotron_mels.npz")
    fix = [g[f"mel_{i:02d}"].astype(np.float32) / np.float32(65535.0) for i in range(16)]
    out = []
    for i in range(n):
        rot = fix[i % 16:] + fix[:i % 16]
        mel = np.concatenate(rot * (frames // sum(m.shape[1] for m in rot) + 1), axis=1)[:, :frames]
        out.append(np.ascontiguousarray(mel))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--frames", type=int, default=800)
    ap.add_argument("--sizes", default="1,8,24,25,64")
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    info = card()
    with contextlib.redirect_stdout(io.StringIO()):
        m = WaveRNN(mode="MOL", **CTOR)
    m.load_state_dict(checkpoint())
    eng = cabi.Engine(m.hot_state(), n_classes=m.n_classes, mode="MOL", precision="fp16", engine="tcgen05")
    eng.attach_upsampler(m.state_dict())
    lib = eng.lib
    hop = CTOR["hop_length"]

    def events():
        return torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    for n in [int(s) for s in a.sizes.split(",")]:
        mels = mels_of(n, a.frames)
        seeds = [11 + i for i in range(n)]
        T = a.frames
        steps, wave_len = T * hop, (T - 1) * hop

        def host():
            e0, e1 = events()
            e0.record()
            wavs = eng.vocode_many_host(mels, seeds, batched=False)
            e1.record()
            torch.cuda.synchronize(dev)
            return e0.elapsed_time(e1) * 1e3 / steps, wavs

        def live_many():
            wavs = [np.full(wave_len, np.nan) for _ in range(n)]
            b, keep = cabi.vocode_batch([(x.ctypes.data, T, s, w.ctypes.data) for x, s, w in zip(mels, seeds, wavs)],
                                        batched=False)
            nr = np.zeros(n, dtype=np.int64)
            first = [None] * n
            e0, e1 = events()
            e0.record()
            t0 = time.perf_counter()
            cabi._check(lib, lib.wrnn_vocode_many_live_start(eng._h, ctypes.byref(b), None))
            e1.record()
            while True:
                rc = lib.wrnn_vocode_many_live_poll(eng._h, 100, nr.ctypes.data)
                now = time.perf_counter() - t0
                for i in np.flatnonzero(nr > 0):
                    if first[i] is None:
                        first[i] = now
                if rc != 1:
                    cabi._check(lib, rc)
                    break
            torch.cuda.synchronize(dev)
            del keep
            return e0.elapsed_time(e1) * 1e3 / steps, wavs, first

        def live_one():
            wav = np.full(wave_len, np.nan)
            job = cabi.WrnnVocodeJob(mels[0].ctypes.data, T, 0, 0, 0, 0, seeds[0], wav.ctypes.data)
            nr = ctypes.c_int64(0)
            e0, e1 = events()
            e0.record()
            cabi._check(lib, lib.wrnn_vocode_live_start(eng._h, ctypes.byref(job), None))
            e1.record()
            while True:
                rc = lib.wrnn_vocode_live_poll(eng._h, 100, ctypes.byref(nr))
                if rc != 1:
                    cabi._check(lib, rc)
                    break
            torch.cuda.synchronize(dev)
            return e0.elapsed_time(e1) * 1e3 / steps, wav

        host()                                           # warm-up: modules, scratch, pinned buffer
        live_many()
        if n == 1:
            live_one()
        t_host, t_live, t_one, firsts = [], [], [], []
        for _ in range(a.runs):
            th, want = host()
            tl, got, first = live_many()
            for g_, w_ in zip(got, want):
                assert np.array_equal(g_.view(np.int64), w_.view(np.int64)), "live waveform differs from vocode_many_host's"
            t_host.append(th)
            t_live.append(tl)
            firsts += first
            if n == 1:
                to, got1 = live_one()
                assert np.array_equal(got1.view(np.int64), want[0].view(np.int64)), "wrnn_vocode_live_start differs"
                t_one.append(to)
        us_live, us_host = statistics.median(t_live), statistics.median(t_host)
        res = dict(engine=eng.name, utterances=n, frames=T, steps=steps, runs=a.runs,
                   us_per_step_live=[round(x, 3) for x in t_live], us_per_step_vocode_many_host=[round(x, 3) for x in t_host],
                   live_over_host=round(us_live / us_host, 4),
                   first_audio_ms_median=round(statistics.median(firsts) * 1e3, 3),
                   first_audio_ms_max=round(max(firsts) * 1e3, 3),
                   real_time_factor_per_stream=round(1e6 / CTOR["sample_rate"] / us_live, 2), bit_identical=True)
        if n == 1:
            res["us_per_step_vocode_live_start"] = [round(x, 3) for x in t_one]
            res["live_many_over_live_start"] = round(us_live / statistics.median(t_one), 4)
        print(json.dumps(dict(res, **info)), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
