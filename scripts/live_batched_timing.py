"""Times 10 s utterances arriving staggered at one server, served three ways, on the shipped LJSpeech checkpoint, fp16,
persistent engine, and writes one JSON line per way to --out/live_batched_timing.jsonl (and stdout), each with the card it
ran on (name, power limit, maximum SM clock from nvidia-smi):

  batched:    a live session of --capacity slots; each arrival is submitted with wrnn_live_submit_batched at the default
              geometry (target 11000, overlap 550: 20 folds of 12,100 steps for 802 frames).
  unbatched:  the same session, each arrival submitted with wrnn_live_submit (one fold of 220,275 steps).
  many_host:  closed jobs of wrnn_vocode_many_host (batched, the same geometry): each job takes every arrival that is
              waiting when the previous job returns, and its waveforms arrive all at once when it returns.

Per arrival: first audio (arrival to the first n_ready > 0; many_host: to its job's return) and completion (arrival to
the whole waveform).  us per step: live, the host clock over the samples of a ticket's leading fold delivered between
polls (100 us) while the prefix grows one sample per step, median over tickets; many_host, each job's time over its
12,100 steps.  Every waveform is checked bit-identical to wrnn_vocode_host's.

    python scripts/live_batched_timing.py --out DIR [--arrivals 4] [--gap-ms 100] [--frames 802] [--capacity 64]"""
import argparse
import contextlib
import io
import json
import statistics
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "scripts"))

from live_many_timing import mels_of  # noqa: E402
from live_timing import CTOR, card, checkpoint  # noqa: E402
from wavernn_b200 import WaveRNN, cabi  # noqa: E402

TARGET, OVERLAP = 11000, 550


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--arrivals", type=int, default=4)
    ap.add_argument("--gap-ms", type=float, default=100.0)
    ap.add_argument("--frames", type=int, default=802)
    ap.add_argument("--capacity", type=int, default=64)
    a = ap.parse_args()
    out = Path(a.out)
    out.mkdir(parents=True, exist_ok=True)
    log = open(out / "live_batched_timing.jsonl", "w")
    info = card()

    def emit(d):
        line = json.dumps(dict(d, **info))
        print(line, flush=True)
        log.write(line + "\n")
        log.flush()

    with contextlib.redirect_stdout(io.StringIO()):
        m = WaveRNN(mode="MOL", **CTOR)
    m.load_state_dict(checkpoint())
    eng = cabi.Engine(m.hot_state(), n_classes=m.n_classes, mode="MOL", precision="fp16", engine="tcgen05")
    eng.attach_upsampler(m.state_dict())
    hop, T, n = CTOR["hop_length"], a.frames, a.arrivals
    wave_len, stride = (T - 1) * hop, TARGET + OVERLAP
    mels, seeds = mels_of(n, T), [21 + i for i in range(n)]
    gap = a.gap_ms / 1e3
    want = {}

    def reference(i, batched):
        if (i, batched) not in want:
            want[(i, batched)] = eng.vocode_host(mels[i], batched=batched, target=TARGET, overlap=OVERLAP, philox_seed=seeds[i])
        return want[(i, batched)]

    def live(batched):
        first, done, marks, tks = {}, {}, {}, []
        with eng.live_session(a.capacity, T) as s:
            def poll():
                s.poll_once(100)
                now = time.perf_counter()
                for i, t in enumerate(tks):
                    p = s._prev[t]
                    if i not in first and p > 0:
                        first[i] = now
                    if i not in done and s.states[t] != cabi.LIVE_RUNNING:
                        done[i] = now
                    if 0 < p < (stride if batched else wave_len):
                        marks.setdefault(i, []).append((now, p))
            t0 = time.perf_counter()
            arrive = [t0 + k * gap for k in range(n)]
            for i in range(n):
                while time.perf_counter() < arrive[i]:
                    poll()
                while True:
                    try:
                        tks.append(s.submit_batched(mels[i], philox_seed=seeds[i], target=TARGET, overlap=OVERLAP)
                                   if batched else s.submit(mels[i], philox_seed=seeds[i]))
                        break
                    except cabi.EngineError as e:
                        if e.code != cabi.WRNN_E_BUSY:
                            raise
                        poll()
            while len(done) < n:
                poll()
            for i, t in enumerate(tks):
                assert np.array_equal(s.waves[t].view(np.int64), reference(i, batched).view(np.int64)), "waveform differs"
        per = [(mk[-1][0] - mk[0][0]) * 1e6 / (mk[-1][1] - mk[0][1]) for mk in marks.values()
               if len(mk) > 1 and mk[-1][1] > mk[0][1]]
        return ([(first[i] - arrive[i]) * 1e3 for i in range(n)], [(done[i] - arrive[i]) * 1e3 for i in range(n)],
                statistics.median(per) if per else None)

    def many_host():
        t0 = time.perf_counter()
        arrive = [t0 + k * gap for k in range(n)]
        done, steps_us, nxt = {}, [], 0
        while nxt < n:
            while time.perf_counter() < arrive[nxt]:
                time.sleep(1e-4)
            now = time.perf_counter()
            job = [i for i in range(nxt, n) if arrive[i] <= now]
            j0 = time.perf_counter()
            wavs = eng.vocode_many_host([mels[i] for i in job], [seeds[i] for i in job], batched=True, target=TARGET,
                                        overlap=OVERLAP)
            j1 = time.perf_counter()
            steps_us.append((j1 - j0) * 1e6 / (TARGET + 2 * OVERLAP))
            for i, w in zip(job, wavs):
                done[i] = j1
                assert np.array_equal(w.view(np.int64), reference(i, True).view(np.int64)), "waveform differs"
            nxt = job[-1] + 1
        lat = [(done[i] - arrive[i]) * 1e3 for i in range(n)]
        return lat, lat, statistics.median(steps_us)

    for i in range(n):                                   # the references first: no other call runs while a session is open
        reference(i, True), reference(i, False)
    live(True)                                           # warm-up of every path
    live(False)
    many_host()
    for way, run in [("batched", lambda: live(True)), ("unbatched", lambda: live(False)), ("many_host", many_host)]:
        first, done, us = run()
        emit(dict(measure=way, frames=T, arrivals=n, gap_ms=a.gap_ms, capacity=a.capacity,
                  first_audio_ms=[round(x, 2) for x in first], first_audio_ms_median=round(statistics.median(first), 2),
                  complete_ms=[round(x, 2) for x in done], complete_ms_median=round(statistics.median(done), 2),
                  complete_ms_max=round(max(done), 2), us_per_step=None if us is None else round(us, 3),
                  bit_identical=True))
    eng.close()


if __name__ == "__main__":
    main()
