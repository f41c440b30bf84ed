"""Times live sessions (wrnn_live_*) on the shipped LJSpeech checkpoint, fp16, persistent engine, and writes one JSON line
per measurement to --out/live_session_timing.jsonl (and stdout), each with the card it ran on (name, power limit, maximum
SM clock from nvidia-smi).

  step:      a session of C slots holding C utterances of --frames frames (submitted back to back, so admitted at
             successive boundaries), against wrnn_vocode_many_live of the same C mels, alternating, --runs of each.
             Session us per step: host clock over each ticket's samples delivered while every slot was held (polls of
             100 us), median over tickets; vocode_many_live's the same way.
  join:      C - 1 utterances mid-way, then one more submitted: submit to its first n_ready > 0 (conditioning network on
             the spare SMs, posting, admission at the next boundary, first 64 samples).  Against today's alternative:
             what the running job has left, plus a new job's first audio.
  cond:      wrnn_conditioning_frames of an --frames mel on an idle device (CUDA events), for reference.
  mix:       Tacotron fixture mels arriving at seeded exponential gaps at --rates arrivals per second, --arrivals each, at
             capacity 24 and 64: per listener the real-time factor (its audio over submit-to-complete) and the admission
             latency (submit to first audio).  Every waveform is checked bit-identical to wrnn_vocode_host's.

    python scripts/live_session_timing.py --out DIR [--runs 2] [--frames 800] [--sizes 1,24,25,64]"""
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

from live_many_timing import mels_of  # noqa: E402
from live_timing import CTOR, GOLDEN, card, checkpoint  # noqa: E402
from wavernn_b200 import WaveRNN, cabi  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--frames", type=int, default=800)
    ap.add_argument("--sizes", default="1,24,25,64")
    ap.add_argument("--rates", default="5,20")
    ap.add_argument("--arrivals", type=int, default=40)
    a = ap.parse_args()
    out = Path(a.out)
    out.mkdir(parents=True, exist_ok=True)
    log = open(out / "live_session_timing.jsonl", "w")
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
    hop, sr = CTOR["hop_length"], CTOR["sample_rate"]
    T = a.frames
    wave_len = (T - 1) * hop

    def session_step(C, mels, seeds):
        """us per step of a session holding C utterances, from each ticket's samples delivered while all were held."""
        with eng.live_session(C, T) as s:
            tks = [s.submit(x, philox_seed=sd) for x, sd in zip(mels, seeds)]
            marks = {t: [] for t in tks}
            rc = 1
            while rc == 1:
                rc, _ = s.poll_once(100)
                now = time.perf_counter()
                full = all(s._prev[t] > 0 for t in tks) and all(s._prev[t] < wave_len for t in tks)
                if full:
                    for t in tks:
                        marks[t].append((now, s._prev[t]))
            per = [(mk[-1][0] - mk[0][0]) * 1e6 / (mk[-1][1] - mk[0][1]) for mk in marks.values() if len(mk) > 1 and mk[-1][1] > mk[0][1]]
            return statistics.median(per), [s.waves[t] for t in tks]

    def many_live(mels, seeds):
        """The same measure for wrnn_vocode_many_live of the same mels."""
        lib, n = eng.lib, len(mels)
        wavs = [np.full(wave_len, np.nan) for _ in range(n)]
        b, keep = cabi.vocode_batch([(x.ctypes.data, T, sd, w.ctypes.data) for x, sd, w in zip(mels, seeds, wavs)],
                                    batched=False)
        cabi._check(lib, lib.wrnn_vocode_many_live_start(eng._h, ctypes.byref(b), None))
        nr = np.zeros(n, dtype=np.int64)
        marks = [[] for _ in range(n)]
        rc = 1
        while rc == 1:
            rc = lib.wrnn_vocode_many_live_poll(eng._h, 100, nr.ctypes.data)
            now = time.perf_counter()
            if nr.min() > 0 and nr.max() < wave_len:
                for i in range(n):
                    marks[i].append((now, int(nr[i])))
        cabi._check(lib, min(rc, 0))
        del keep
        per = [(mk[-1][0] - mk[0][0]) * 1e6 / (mk[-1][1] - mk[0][1]) for mk in marks if len(mk) > 1 and mk[-1][1] > mk[0][1]]
        return statistics.median(per), wavs

    for C in [int(x) for x in a.sizes.split(",")]:
        mels = mels_of(C, T)
        seeds = [11 + i for i in range(C)]
        session_step(C, mels, seeds)                         # warm-up
        t_ses, t_many = [], []
        for _ in range(a.runs):
            us, got = session_step(C, mels, seeds)
            t_ses.append(us)
            us, want = many_live(mels, seeds)
            t_many.append(us)
            for g_, w_ in zip(got, want):
                assert np.array_equal(g_.view(np.int64), w_.view(np.int64)), "session waveform differs from vocode_many_live's"
        emit(dict(measure="step", capacity=C, frames=T, runs=a.runs, us_per_step_session=[round(x, 3) for x in t_ses],
                  us_per_step_vocode_many_live=[round(x, 3) for x in t_many],
                  session_over_many_live=round(statistics.median(t_ses) / statistics.median(t_many), 4), bit_identical=True))

        # join: C - 1 mid-utterance, then one more
        if C > 1:
            with eng.live_session(C, T) as s:
                tks = [s.submit(x, philox_seed=sd) for x, sd in zip(mels[:C - 1], seeds[:C - 1])]
                while min(s._prev[t] for t in tks) < wave_len // 3:
                    s.poll_once(100)
                joins = []
                for k in range(3):
                    t0 = time.perf_counter()
                    j = s.submit(mels[-1][:, :100], philox_seed=99 + k)
                    while s._prev[j] == 0:
                        s.poll_once(50)
                    joins.append((time.perf_counter() - t0) * 1e3)
                    while s.states[j] == cabi.LIVE_RUNNING:
                        s.poll_once(100)
                left = min(wave_len - s._prev[t] for t in tks)
                us_step = statistics.median(t_ses)
                s.close()
            emit(dict(measure="join", capacity=C, first_audio_ms=[round(x, 3) for x in joins],
                      first_audio_ms_median=round(statistics.median(joins), 3), first_audio_ms_max=round(max(joins), 3),
                      wait_for_running_job_ms_at_least=round(left * us_step / 1e3, 1)))

    # conditioning network of one mel, idle device
    mel = torch.from_numpy(mels_of(1, T)[0]).cuda()
    mf = torch.empty((T + 4) * 80, device="cuda")
    af = torch.empty(T * 128, device="cuda")
    ts = []
    for _ in range(5):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        eng.conditioning_frames(mel=mel.data_ptr(), T=T, mel_frames=mf.data_ptr(), aux_frames=af.data_ptr(),
                                stream=torch.cuda.current_stream().cuda_stream)
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    emit(dict(measure="cond", frames=T, ms_idle=round(statistics.median(ts[1:]), 3)))

    # sustained mix of the fixture mels
    g = np.load(GOLDEN / "tacotron_mels.npz")
    fix = [np.ascontiguousarray(g[f"mel_{i:02d}"].astype(np.float32) / np.float32(65535.0)) for i in range(16)]
    max_T = max(x.shape[1] for x in fix)
    for C in (24, 64):
        for rate in [float(r) for r in a.rates.split(",")]:
            rs = np.random.RandomState(7)
            gaps = rs.exponential(1.0 / rate, size=a.arrivals)
            pick = rs.randint(0, 16, size=a.arrivals)
            sub, first, done, tk_of = {}, {}, {}, []
            with eng.live_session(C, max_T) as s:
                t0 = time.perf_counter()
                due = t0
                for k in range(a.arrivals):
                    due += gaps[k]
                    while time.perf_counter() < due:
                        s.poll_once(100)
                        now = time.perf_counter()
                        for t in tk_of:
                            if t not in first and s._prev[t] > 0:
                                first[t] = now
                            if t not in done and s.states[t] != cabi.LIVE_RUNNING:
                                done[t] = now
                    while True:
                        try:
                            t = s.submit(fix[pick[k]], philox_seed=1000 + k)
                            break
                        except cabi.EngineError as e:
                            if e.code != cabi.WRNN_E_BUSY:
                                raise
                            s.poll_once(100)
                    sub[t] = time.perf_counter()
                    tk_of.append(t)
                rc = 1
                while rc == 1:
                    rc, _ = s.poll_once(100)
                    now = time.perf_counter()
                    for t in tk_of:
                        if t not in first and s._prev[t] > 0:
                            first[t] = now
                        if t not in done and s.states[t] != cabi.LIVE_RUNNING:
                            done[t] = now
                waves = {t: s.waves[t] for t in tk_of}
            for k, t in enumerate(tk_of[:4]):
                want = eng.vocode_host(fix[pick[k]], batched=False, philox_seed=1000 + k)
                assert np.array_equal(waves[t].view(np.int64), want.view(np.int64)), "mix waveform differs"
            rtf = [waves[t].size / sr / (done[t] - sub[t]) for t in tk_of]
            adm = [(first[t] - sub[t]) * 1e3 for t in tk_of]
            emit(dict(measure="mix", capacity=C, arrivals_per_s=rate, arrivals=a.arrivals,
                      rtf_per_listener_median=round(statistics.median(rtf), 2), rtf_per_listener_min=round(min(rtf), 2),
                      admission_ms_median=round(statistics.median(adm), 2), admission_ms_max=round(max(adm), 2)))
    eng.close()


if __name__ == "__main__":
    main()
