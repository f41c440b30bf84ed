"""Live sessions (wrnn_live_open / _submit / _cancel / _poll / _close) on the device: utterances submitted at any time
are admitted into the running persistent kernel, and every delivered waveform is bit-identical to its own unbatched
wrnn_vocode_host, whatever its slot, its admission step, the launch that served it and whatever else was in flight."""
import ctypes
import time

import numpy as np
import pytest

import helpers
from wavernn_b200 import cabi

pytestmark = pytest.mark.gpu

HOP = 275


@pytest.fixture(scope="module")
def lib():
    if not cabi.is_built():
        import __graft_entry__ as g
        g.build()
    return cabi.load()


def _engine(model, precision="fp16", engine="tcgen05"):
    eng = cabi.Engine(model.hot_state(), n_classes=model.n_classes, mode=model.mode, precision=precision, engine=engine)
    eng.attach_upsampler(model.state_dict())
    return eng


def _mels(Ts, seed):
    return [np.ascontiguousarray(helpers.make_mel(T, seed=seed + i)[0].numpy()) for i, T in enumerate(Ts)]


def _same(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.int64), b.view(np.int64))


def _submit(sess, mel, seed):
    """Submits, polling while every slot is held."""
    while True:
        try:
            return sess.submit(mel, philox_seed=seed)
        except cabi.EngineError as e:
            if e.code != cabi.WRNN_E_BUSY:
                raise
            sess.poll_once(1000)


def _drain(sess):
    rc = 1
    while rc == 1:
        rc, _ = sess.poll_once(1000)


def _staggered(sess, jobs, lead=1):
    """Submits jobs [(mel, seed)] one by one, each once the previous ticket has delivered `lead` samples or more (so
    that it joins a running launch), then drains.  Returns the tickets."""
    tickets = []
    for mel, seed in jobs:
        if tickets:
            while sess._prev[tickets[-1]] < lead and sess.states[tickets[-1]] == cabi.LIVE_RUNNING:
                sess.poll_once(1000)
        tickets.append(_submit(sess, mel, seed))
    _drain(sess)
    return tickets


@pytest.mark.parametrize("mode,precision,mu_law,capacity", [
    ("MOL", "fp16", False, 1), ("MOL", "fp16", False, 64), ("MOL", "bf16", False, 24), ("MOL", "bf16", False, 25),
    ("RAW", "fp16", True, 24), ("RAW", "fp16", True, 25), ("RAW", "bf16", False, 1), ("RAW", "bf16", False, 64)])
def test_session_equals_vocode_host(lib, mode, precision, mu_law, capacity):
    """Every session kernel (MoL / RAW x fp16 / bf16 x small / BIG tile), staggered admissions of mixed lengths, more
    utterances than slots at capacity 1."""
    m = helpers.make_model(0, mode)
    eng = _engine(m, precision)
    Ts = [40, 26, 61] if capacity > 1 else [30, 22, 41]
    mels, seeds = _mels(Ts, 10), [1234, 7, 2**40 + 3]
    with eng.live_session(capacity, 64, mu_law=mu_law) as sess:
        tickets = _staggered(sess, list(zip(mels, seeds)))
        waves = [sess.waves[t] for t in tickets]
        assert all(sess.states[t] == cabi.LIVE_DONE for t in tickets)
    assert eng.name.startswith("tcgen05")
    for mel, seed, w in zip(mels, seeds, waves):
        assert _same(w, eng.vocode_host(mel, batched=False, mu_law=mu_law, philox_seed=seed))


def test_admission_into_a_running_launch(lib):
    """Listeners join while earlier ones are mid-utterance: no new launch, the same utterance admitted at two different
    steps (and slots) gives the same bits, and slots are reused by utterances of mixed lengths."""
    m = helpers.make_model(0, "MOL")
    eng = _engine(m)
    mels = _mels([300, 45, 80, 33, 52], 30)
    with eng.live_session(3, 300) as sess:
        first = sess.submit(mels[0], philox_seed=5)
        while sess._prev[first] == 0:
            sess.poll_once(1000)
        launches = eng.launch_count
        late = []
        for i, seed in [(1, 6), (2, 7), (1, 6), (3, 8), (4, 9), (2, 7)]:
            while late and sess._prev[late[-1]] == 0 and sess.states[late[-1]] == cabi.LIVE_RUNNING:
                sess.poll_once(1000)
            late.append(_submit(sess, mels[i], seed))
            assert sess.states[first] == cabi.LIVE_RUNNING
        joined = eng.launch_count == launches
        _drain(sess)
        print(f"launches during the joins: {eng.launch_count - launches}")
        assert joined, "a listener that arrived mid-utterance started a new launch"
        w = {t: sess.waves[t] for t in [first] + late}
    assert _same(w[late[0]], w[late[2]]) and _same(w[late[1]], w[late[5]])
    for t, (i, seed) in zip([first] + late, [(0, 5), (1, 6), (2, 7), (1, 6), (3, 8), (4, 9), (2, 7)]):
        assert _same(w[t], eng.vocode_host(mels[i], batched=False, philox_seed=seed)), t


def test_cancel_mid_utterance_and_reuse_the_slot(lib):
    m = helpers.make_model(0, "RAW")
    eng = _engine(m, "bf16")
    mels = _mels([400, 30, 35], 50)
    with eng.live_session(2, 400, mu_law=True) as sess:
        a = sess.submit(mels[0], philox_seed=1)
        b = sess.submit(mels[1], philox_seed=2)
        while sess._prev[a] < 2 * 64:
            sess.poll_once(1000)
        sess.cancel(a)
        while sess.states[a] == cabi.LIVE_RUNNING:
            sess.poll_once(1000)
        assert sess.states[a] == cabi.LIVE_CANCELLED
        cut = sess._prev[a]
        assert 0 < cut < sess.waves[a].size
        c = sess.submit(mels[2], philox_seed=3)            # into the slot the cancelled ticket held
        _drain(sess)
        with pytest.raises(cabi.EngineError, match="not in flight"):
            sess.cancel(a)
        got = {t: sess.waves[t] for t in (a, b, c)}
    want_a = eng.vocode_host(mels[0], batched=False, mu_law=True, philox_seed=1)
    assert _same(got[a][:cut], want_a[:cut])
    assert _same(got[b], eng.vocode_host(mels[1], batched=False, mu_law=True, philox_seed=2))
    assert _same(got[c], eng.vocode_host(mels[2], batched=False, mu_law=True, philox_seed=3))


def test_idle_session_exits_and_the_next_submit_relaunches(lib):
    m = helpers.make_model(0, "MOL")
    eng = _engine(m)
    mels = _mels([24, 27], 60)
    with eng.live_session(4, 64) as sess:
        t0 = sess.submit(mels[0], philox_seed=11)
        _drain(sess)
        n0 = eng.launch_count
        time.sleep(0.05)                                   # the launch stops at its next boundary
        t1 = sess.submit(mels[1], philox_seed=12)        # posted, and the kernel relaunched, once its frames are ready
        _drain(sess)
        assert eng.launch_count == n0 + 1, "the ticket after the kernel exited was not served by one new launch"
        w0, w1 = sess.waves[t0], sess.waves[t1]
    assert _same(w0, eng.vocode_host(mels[0], batched=False, philox_seed=11))
    assert _same(w1, eng.vocode_host(mels[1], batched=False, philox_seed=12))


def test_busy_during_a_session_and_refusals(lib):
    m = helpers.make_model(0, "MOL")
    eng = _engine(m)
    short = _mels([26], 70)[0]
    before = eng.vocode_host(short, batched=False, philox_seed=3)
    sess = eng.live_session(2, 100)
    with pytest.raises(cabi.EngineError, match="live session is open") as e:
        eng.live_session(2, 100)
    assert e.value.code == cabi.WRNN_E_BUSY

    def busy(fn, *a, **k):
        with pytest.raises(cabi.EngineError, match="live session is open") as e:
            fn(*a, **k)
        assert e.value.code == cabi.WRNN_E_BUSY
    busy(eng.vocode_host, short, batched=False, philox_seed=3)
    busy(eng.vocode_many_host, [short], [3], batched=False)
    busy(eng.score_many_host, [short], [np.zeros(25 * HOP, np.float32)])
    busy(eng.check)
    busy(lambda: list(eng.vocode_live(short, philox_seed=1)))
    busy(lambda: list(eng.vocode_many_live([short], [1])))
    one = ctypes.c_int64(-1)
    assert lib.wrnn_vocode_live_poll(eng._h, 0, ctypes.byref(one)) == cabi.WRNN_E_INVALID and one.value == -1
    assert b"wrnn_live_poll" in lib.wrnn_last_error()
    n = np.full(2, -1, dtype=np.int64)
    assert lib.wrnn_vocode_many_live_poll(eng._h, 0, n.ctypes.data) == cabi.WRNN_E_INVALID and (n == -1).all()
    with pytest.raises(cabi.EngineError, match="exceeds the session's max_T"):
        sess.submit(_mels([101], 1)[0], philox_seed=0)
    a = sess.submit(_mels([100], 2)[0], philox_seed=0)
    b = sess.submit(short, philox_seed=3)
    with pytest.raises(cabi.EngineError, match="all 2 slots") as e:
        sess.submit(short, philox_seed=4)
    assert e.value.code == cabi.WRNN_E_BUSY
    _drain(sess)
    assert _same(sess.waves[b], before) and sess.states[a] == cabi.LIVE_DONE
    sess.close()
    with pytest.raises(cabi.EngineError, match="no live session is open"):
        sess.submit(short, philox_seed=3)
    assert np.array_equal(eng.vocode_host(short, batched=False, philox_seed=3), before)
    for e_, match in [(_engine(m, "fp16", "stream"), "66 us per step"), (_engine(m, "bf16", "simt"), "SIMT engine")]:
        with pytest.raises(cabi.EngineError, match=match):
            e_.live_session(2, 100)
    with pytest.raises(cabi.EngineError, match="no upsampler attached"):
        cabi.Engine(m.hot_state()).live_session(2, 100)


def test_destroy_with_a_session_open(lib):
    m = helpers.make_model(0, "MOL")
    eng = _engine(m)
    mels = _mels([200, 60], 80)
    sess = eng.live_session(2, 200)
    sess.submit(mels[0], philox_seed=2)
    sess.submit(mels[1], philox_seed=3)
    sess.poll_once(2000)
    eng.close()                                            # closes the session and waits for the kernel
    eng = _engine(m)
    assert np.isfinite(eng.vocode_host(mels[1], batched=False, philox_seed=3)).all()


def test_session_on_the_checkpoint(lib):
    m = helpers.make_model(0, "MOL")
    m.load_state_dict(helpers.pretrained_state_dict())
    eng = _engine(m)
    mels = [np.ascontiguousarray(x) for x in helpers.tacotron_mels()[:4]]
    seeds = [77, 78, 79, 80]
    with eng.live_session(3, max(x.shape[-1] for x in mels)) as sess:
        tickets = _staggered(sess, list(zip(mels, seeds)), lead=4 * 64)
        waves = [sess.waves[t] for t in tickets]
    for mel, seed, w in zip(mels, seeds, waves):
        assert _same(w, eng.vocode_host(mel, batched=False, philox_seed=seed))
        assert np.abs(w).max() > 1e-3
