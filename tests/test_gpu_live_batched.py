"""Batched live tickets (wrnn_live_submit_batched) on the device: each fold of a batched utterance takes a slot of the
running session kernel, and every delivered waveform is bit-identical to its own batched wrnn_vocode_host, whatever its
slots, the boundaries and launches that served its folds and whatever else was in flight."""
import time

import numpy as np
import pytest

import helpers
from oracle import wavernn_oracle as O
from wavernn_b200 import cabi

pytestmark = pytest.mark.gpu

HOP = 275


@pytest.fixture(scope="module")
def lib():
    if not cabi.is_built():
        import __graft_entry__ as g
        g.build()
    return cabi.load()


def _engine(model, precision="fp16"):
    eng = cabi.Engine(model.hot_state(), n_classes=model.n_classes, mode=model.mode, precision=precision, engine="tcgen05")
    eng.attach_upsampler(model.state_dict())
    return eng


def _mels(Ts, seed):
    return [np.ascontiguousarray(helpers.make_mel(T, seed=seed + i)[0].numpy()) for i, T in enumerate(Ts)]


def _same(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.int64), b.view(np.int64))


def _submit(sess, job):
    """Submits job = (mel, seed, geometry or None for unbatched), polling while too few slots are free."""
    mel, seed, geo = job
    while True:
        try:
            if geo is None:
                return sess.submit(mel, philox_seed=seed)
            return sess.submit_batched(mel, philox_seed=seed, target=geo[0], overlap=geo[1])
        except cabi.EngineError as e:
            if e.code != cabi.WRNN_E_BUSY:
                raise
            sess.poll_once(1000)


def _drain(sess):
    rc = 1
    while rc == 1:
        rc, _ = sess.poll_once(1000)


def _want(eng, job, mu_law=False):
    mel, seed, geo = job
    if geo is None:
        return eng.vocode_host(mel, batched=False, mu_law=mu_law, philox_seed=seed)
    return eng.vocode_host(mel, batched=True, target=geo[0], overlap=geo[1], mu_law=mu_law, philox_seed=seed)


def _staggered(sess, jobs, lead=1):
    """Submits each job once the previous ticket has delivered `lead` samples or more (so that it joins a running
    launch), then drains.  Returns the tickets."""
    tickets = []
    for job in jobs:
        if tickets:
            while sess._prev[tickets[-1]] < lead and sess.states[tickets[-1]] == cabi.LIVE_RUNNING:
                sess.poll_once(1000)
        tickets.append(_submit(sess, job))
    _drain(sess)
    return tickets


@pytest.mark.parametrize("mode,precision,mu_law,capacity", [
    ("MOL", "fp16", False, 1), ("MOL", "fp16", False, 64), ("MOL", "bf16", False, 24), ("MOL", "bf16", False, 25),
    ("RAW", "fp16", True, 24), ("RAW", "fp16", True, 25), ("RAW", "bf16", False, 1), ("RAW", "bf16", False, 64)])
def test_batched_tickets_equal_vocode_host(lib, mode, precision, mu_law, capacity):
    """Every session kernel (MoL / RAW x fp16 / bf16 x small / BIG tile), staggered batched tickets of short geometries,
    one with stride % hop != 0 and a last fold past T * hop; at capacity 1, one fold per ticket."""
    m = helpers.make_model(0, mode)
    eng = _engine(m, precision)
    if capacity == 1:
        mels, geos = _mels([22, 21, 22], 10), [(6000, 100), (5000, 400), (5900, 200)]
    else:
        mels, geos = _mels([30, 26, 41], 10), [(2000, 137), (1100, 110), (2200, 220)]
    jobs = [(x, s, g) for x, s, g in zip(mels, [1234, 7, 2**40 + 3], geos)]
    with eng.live_session(capacity, 41 if capacity > 1 else 24, mu_law=mu_law) as sess:
        tickets = _staggered(sess, jobs)
        waves = [sess.waves[t] for t in tickets]
        assert all(sess.states[t] == cabi.LIVE_DONE for t in tickets)
    for job, w in zip(jobs, waves):
        assert _same(w, _want(eng, job, mu_law))


def test_mixed_session(lib):
    """Unbatched and batched tickets submitted staggered into one session of 8 slots: slots are reused after release,
    WRNN_E_BUSY (taking no slot) while too few are free and the same submit succeeding after a release, and every
    waveform bit-identical, the unbatched ones to their unbatched wrnn_vocode_host."""
    m = helpers.make_model(0, "MOL")
    eng = _engine(m)
    mels = _mels([120, 30, 40, 26, 60, 33], 20)
    with eng.live_session(8, 120) as sess:
        first = sess.submit(mels[0], philox_seed=5)
        while sess._prev[first] == 0:
            sess.poll_once(1000)
        a = sess.submit_batched(mels[4], philox_seed=9, target=3000, overlap=300)    # 5 folds: 6 slots held
        with pytest.raises(cabi.EngineError, match="folds: poll until enough are released") as e:
            sess.submit_batched(mels[2], philox_seed=7, target=2200, overlap=220)   # 5 folds, 2 slots free
        assert e.value.code == cabi.WRNN_E_BUSY
        b = sess.submit(mels[3], philox_seed=8)                    # the free slots are untouched by the refusal
        c = sess.submit(mels[5], philox_seed=10)
        while sess.states[a] == cabi.LIVE_RUNNING:
            sess.poll_once(1000)
        d = _submit(sess, (mels[2], 7, (2200, 220)))                # into the released slots, mid-launch
        rest = _staggered(sess, [(mels[1], 6, (2000, 137)), (mels[3], 8, None), (mels[1], 6, (2000, 137)),
                                 (mels[2], 11, (1500, 100))])
        got = {t: sess.waves[t] for t in [first, a, b, c, d] + rest}
        assert all(sess.states[t] == cabi.LIVE_DONE for t in got)
    jobs = {first: (mels[0], 5, None), a: (mels[4], 9, (3000, 300)), b: (mels[3], 8, None), c: (mels[5], 10, None),
            d: (mels[2], 7, (2200, 220)), rest[0]: (mels[1], 6, (2000, 137)), rest[1]: (mels[3], 8, None),
            rest[2]: (mels[1], 6, (2000, 137)), rest[3]: (mels[2], 11, (1500, 100))}
    assert _same(got[rest[0]], got[rest[2]]) and _same(got[b], got[rest[1]])
    for t, job in jobs.items():
        assert _same(got[t], _want(eng, job)), t


def _post_one_fold_per_poll(lib, eng, sess, mel, seed, geo, pause):
    """Submits a batched ticket whose folds are posted one per poll, `pause` seconds apart; returns it once drained."""
    assert lib.wrnn_debug_live_post_limit(eng._h, 1) == 0
    t = sess.submit_batched(mel, philox_seed=seed, target=geo[0], overlap=geo[1])
    while sess.states[t] == cabi.LIVE_RUNNING:
        sess.poll_once(0)
        time.sleep(pause)
    return t


def test_folds_of_one_ticket_at_different_boundaries_and_launches(lib):
    """Folds posted one per poll: with an unbatched ticket keeping the launch alive, each fold is admitted at a later
    boundary of the same launch; in an otherwise idle session, each fold's launch exits before the next fold is posted,
    so every fold is served by a launch of its own.  The waveforms stay bit-identical to wrnn_vocode_host's."""
    m = helpers.make_model(0, "MOL")
    eng = _engine(m)
    mels = _mels([300, 21, 23], 95)
    geo = (1000, 100)                                          # 6 folds of 1,200 steps for 21 frames
    assert O.fold_geometry(21 * HOP, *geo)[0] == 6
    with eng.live_session(8, 300) as sess:
        keep = sess.submit(mels[0], philox_seed=1)
        while sess._prev[keep] == 0:
            sess.poll_once(1000)
        n0 = eng.launch_count
        a = _post_one_fold_per_poll(lib, eng, sess, mels[1], 2, geo, 0.005)   # 5 ms: several 64-step boundaries apart
        joined = eng.launch_count == n0
        sess.cancel(keep)
        _drain(sess)
        time.sleep(0.05)                                       # the idle launch stops at its next boundary
        n1 = eng.launch_count
        b = _post_one_fold_per_poll(lib, eng, sess, mels[1], 3, geo, 0.1)     # 100 ms: each fold's launch has exited
        launches = eng.launch_count - n1
        c = _post_one_fold_per_poll(lib, eng, sess, mels[2], 4, (2000, 137), 0.1)
        got = {t: sess.waves[t] for t in (a, b, c)}
    print(f"launches for the 6 folds posted 100 ms apart: {launches}")
    assert joined, "the folds posted while a launch ran started a new launch"
    assert launches == 6
    assert _same(got[a], _want(eng, (mels[1], 2, geo)))
    assert _same(got[b], _want(eng, (mels[1], 3, geo)))
    assert _same(got[c], _want(eng, (mels[2], 4, (2000, 137))))


def test_cancel_a_batched_ticket_mid_run(lib):
    m = helpers.make_model(0, "RAW")
    eng = _engine(m, "bf16")
    mels = _mels([300, 30, 35], 50)
    with eng.live_session(10, 300, mu_law=True) as sess:
        a = sess.submit_batched(mels[0], philox_seed=1, target=11000, overlap=550)   # 8 folds
        b = sess.submit(mels[1], philox_seed=2)
        while sess._prev[a] < 2 * 64:
            sess.poll_once(1000)
        sess.cancel(a)
        while sess.states[a] == cabi.LIVE_RUNNING:
            sess.poll_once(1000)
        assert sess.states[a] == cabi.LIVE_CANCELLED
        cut = sess._prev[a]
        assert 0 < cut < sess.waves[a].size
        c = sess.submit_batched(mels[2], philox_seed=3, target=2000, overlap=137)    # into the released slots
        _drain(sess)
        with pytest.raises(cabi.EngineError, match="not in flight"):
            sess.cancel(a)
        got = {t: sess.waves[t] for t in (a, b, c)}
    want_a = eng.vocode_host(mels[0], batched=True, target=11000, overlap=550, mu_law=True, philox_seed=1)
    assert _same(got[a][:cut], want_a[:cut])
    assert _same(got[b], eng.vocode_host(mels[1], batched=False, mu_law=True, philox_seed=2))
    assert _same(got[c], eng.vocode_host(mels[2], batched=True, target=2000, overlap=137, mu_law=True, philox_seed=3))


def test_ten_seconds_at_the_default_geometry_streams_before_completion(lib):
    """A 10 s mel (802 frames, 20 folds at target 11000, overlap 550): n_ready never decreases, and polls see a prefix
    that has started but not finished."""
    m = helpers.make_model(0, "MOL")
    eng = _engine(m)
    mel = _mels([802], 90)[0]
    assert O.fold_geometry(802 * HOP, 11000, 550)[0] == 20
    with eng.live_session(20, 802) as sess:
        t = sess.submit_batched(mel, philox_seed=4)
        seen, rc = [], 1
        while rc == 1:
            rc, _ = sess.poll_once(500)
            seen.append(sess._prev[t])
        w = sess.waves[t]
    wave_len = 801 * HOP
    print(f"polls: {len(seen)}, partial prefixes seen: {sum(0 < s < wave_len for s in seen)}")
    assert seen == sorted(seen) and seen[-1] == wave_len
    assert any(0 < s < wave_len for s in seen)
    assert _same(w, eng.vocode_host(mel, batched=True, target=11000, overlap=550, philox_seed=4))


def test_refusals_leave_the_session_usable(lib):
    m = helpers.make_model(0, "MOL")
    eng = _engine(m)
    mel = _mels([60], 70)[0]
    with eng.live_session(4, 60) as sess:
        with pytest.raises(cabi.EngineError, match="has 9 folds, more than the session's 4 slots") as e:
            sess.submit_batched(mel, philox_seed=1, target=2000, overlap=50)
        assert e.value.code == cabi.WRNN_E_INVALID
        with pytest.raises(cabi.EngineError, match="16500 samples exceed a slot's row of .* = 16225"):
            sess.submit_batched(mel, philox_seed=1, target=15000, overlap=750)
        with pytest.raises(cabi.EngineError, match="target > 0 and overlap > 0"):
            sess.submit_batched(mel, philox_seed=1, target=2000, overlap=0)
        with pytest.raises(cabi.EngineError, match="exceeds the session's max_T"):
            sess.submit_batched(_mels([61], 1)[0], philox_seed=1, target=2000, overlap=137)
        t = sess.submit_batched(mel, philox_seed=1, target=6000, overlap=300)    # 3 folds
        _drain(sess)
        w = sess.waves[t]
    assert _same(w, eng.vocode_host(mel, batched=True, target=6000, overlap=300, philox_seed=1))


def test_batched_session_on_the_checkpoint(lib):
    m = helpers.make_model(0, "MOL")
    m.load_state_dict(helpers.pretrained_state_dict())
    eng = _engine(m)
    mels = [np.ascontiguousarray(x) for x in helpers.tacotron_mels()[:3]]
    seeds = [77, 78, 79]
    with eng.live_session(64, max(x.shape[-1] for x in mels)) as sess:
        tickets = _staggered(sess, [(x, s, (11000, 550)) for x, s in zip(mels, seeds)], lead=4 * 64)
        waves = [sess.waves[t] for t in tickets]
    for mel, seed, w in zip(mels, seeds, waves):
        assert _same(w, eng.vocode_host(mel, batched=True, target=11000, overlap=550, philox_seed=seed))
        assert np.abs(w).max() > 1e-3
