"""Host-side pieces of live unbatched vocoding (wrnn_vocode_live_start / _poll), checked without a device: the epilogue
each poll applies to the newly published samples (through the wrnn_debug_live_epilogue hook) against the reference's
host epilogue and a restatement of wrnn_epilogue_kernel, and the refusals that need no handle."""
import ctypes
import math
import sys

import numpy as np
import pytest

import helpers
from wavernn_b200 import cabi, vocoder
from wavernn_b200.sharding import unbatched_geometry

HOP = 275
T = 30                                   # 8,250 generated samples, 7,975 in the waveform, the last 5,500 faded out
L, WAVE = T * HOP, (T - 1) * HOP
TAIL0 = WAVE - 20 * HOP                  # first sample of the fade-out


@pytest.fixture(scope="module")
def lib():
    if not cabi.is_built():
        import __graft_entry__ as g
        g.build()
    return cabi.load()


def _live(lib, x, mu_law, n_classes, n=WAVE):
    wav = np.full(max(n, 1), np.nan)
    x = np.ascontiguousarray(x, dtype=np.float32)
    assert lib.wrnn_debug_live_epilogue(x.ctypes.data, n, WAVE, HOP, int(mu_law), n_classes, wav.ctypes.data) == 0
    return wav[:n]


def _mu_table(lib, n_classes):
    mu = np.empty(n_classes)
    assert lib.wrnn_debug_epilogue_tables(0, 1, n_classes, HOP, None, None, mu.ctypes.data, None) == 0
    return mu


def _kernel_restatement(lib, x, mu_law, n_classes):
    """wrnn_epilogue_kernel in the unbatched geometry, in numpy: the label from the fp32 expression rounded half to even
    (saturating, then clamped), v = 0.0 + y, then the fade-out."""
    f = np.float32
    x = x.astype(f)
    y = x[:WAVE].astype(np.float64)
    if mu_law:
        r = np.rint((x[:WAVE] + f(1)) * (f(0.5) * f(n_classes - 1)))
        assert r.dtype == f
        lbl = np.where(np.isnan(r), 0, np.clip(r, 0, n_classes - 1)).astype(np.int64)
        y = _mu_table(lib, n_classes)[lbl]
    v = np.float64(0.0) + y
    v[TAIL0:] = v[TAIL0:] * np.linspace(1, 0, 20 * HOP)
    return v


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


def _specials(n_classes):
    """-0.0, +-1, values just outside [-1, 1], exact labels and fp32 values whose label expression lands exactly on a
    midpoint k + 0.5 (rounded half to even: both parities of k)."""
    f = np.float32
    out = [f(-0.0), f(0.0), f(1), f(-1), np.nextafter(f(1), f(2)), np.nextafter(f(-1), f(-2)), f(1.5), f(-1.5)]
    k = np.arange(n_classes, dtype=f)
    out += list(f(2) * k / (f(n_classes) - f(1)) - f(1))
    mids = []
    for kk in range(n_classes - 1):
        c = f((kk + 0.5) / (0.5 * (n_classes - 1)) - 1.0)
        for d in range(-4, 5):
            xf = c
            for _ in range(abs(d)):
                xf = np.nextafter(xf, f(np.sign(d) * 2))
            if (xf + f(1)) * (f(0.5) * f(n_classes - 1)) == f(kk + 0.5):
                mids.append(xf)
                break
    assert len(mids) > n_classes // 4 and {int(np.rint((m + f(1)) * f(0.5 * (n_classes - 1)))) % 2 for m in mids} == {0}
    return np.array(out + mids, dtype=f), np.array(mids, dtype=f)


def _samples(rs, specials, labels_only, n_classes):
    """A whole generated fold (L samples), the special values placed both before and inside the fade-out."""
    f = np.float32
    if labels_only:
        x = f(2) * rs.randint(0, n_classes, size=L).astype(f) / (f(n_classes) - f(1)) - f(1)
    else:
        x = rs.uniform(-1, 1, size=L).astype(f)
    m = len(specials)
    assert 2 * m < 20 * HOP and m < TAIL0
    x[100:100 + m] = specials
    x[TAIL0 + 7:TAIL0 + 7 + m] = specials
    x[WAVE - m:WAVE] = specials                       # the last samples of the waveform
    return x


def _scalar_decode_mu_law(y, mu, from_labels):
    """decode_mu_law evaluated with the C library's pow, as the library's table is (tests/test_vocode_abi.py)."""
    assert not from_labels
    n = mu - 1
    return np.array([np.sign(v) / n * (math.pow(1 + n, abs(v)) - 1) for v in np.ravel(y)]).reshape(np.shape(y))


@pytest.mark.parametrize("mode,mu_law", [("MOL", False), ("RAW", False), ("RAW", True)])
def test_live_epilogue_is_the_device_epilogue(lib, mode, mu_law):
    n_classes = 30 if mode == "MOL" else 512
    specials, mids = _specials(n_classes if mode == "RAW" else 512)
    rs = np.random.RandomState(11)
    x = _samples(rs, specials, mode == "RAW" and mu_law, n_classes)
    got = _live(lib, x, mu_law, n_classes)
    want = _kernel_restatement(lib, x, mu_law, n_classes)
    assert np.array_equal(_bits(got), _bits(want))
    if not mu_law:                   # -0.0 becomes +0.0 (0.0 + y), as on the device; the rest passes through
        neg0 = 100 + np.flatnonzero(np.signbit(specials) & (specials == 0))
        assert len(neg0) == 1 and _bits(got[neg0])[0] == 0
        assert np.array_equal(got[100:100 + len(specials)], specials.astype(np.float64))
    else:
        mu = _mu_table(lib, n_classes)
        outside = 100 + np.flatnonzero(np.abs(specials) > 1)
        assert set(got[outside]) == {mu[0], mu[-1]}
        # exact midpoints round half to even
        at = 100 + len(specials) - len(mids) + np.arange(len(mids))
        lbl = np.rint((mids + np.float32(1)) * np.float32(0.5 * (n_classes - 1))).astype(np.int64)
        assert np.all(lbl % 2 == 0) and np.array_equal(got[at], mu[lbl])
    # every prefix a poll can deliver is the prefix of the whole
    for n in (0, 1, 63, 64, TAIL0, TAIL0 + 1, WAVE - 1):
        assert np.array_equal(_bits(_live(lib, x, mu_law, n_classes, n)), _bits(got[:n]))


@pytest.mark.parametrize("mode,mu_law", [("MOL", False), ("RAW", False), ("RAW", True)])
def test_live_epilogue_equals_reference_host_epilogue(lib, monkeypatch, mode, mu_law):
    """Against vocoder.py::_epilogue (the reference's :243-258) in the unbatched geometry, on the samples the kernels can
    write: any fp32 value for MoL, the labels x_k = 2k/(n-1) - 1 for RAW (never -0.0).  Equal as numbers (the reference keeps a -0.0
    sample's sign, the device epilogue does not); with mu-law, decode_mu_law is evaluated with the C library's pow, as
    the library's table is."""
    m = helpers.make_model(0, mode)
    if mu_law:
        monkeypatch.setattr(vocoder, "decode_mu_law", _scalar_decode_mu_law)
    specials, _ = _specials(m.n_classes if mode == "RAW" else 512)
    if mode == "RAW":
        specials = specials[(specials >= -1) & (specials <= 1)]
        f = np.float32
        k = np.rint((specials + f(1)) * f(0.5 * (m.n_classes - 1))).astype(np.int64)
        specials = (f(2) * k.astype(f) / (f(m.n_classes) - f(1)) - f(1)).astype(f)
    x = _samples(np.random.RandomState(5), specials, mode == "RAW", m.n_classes)
    got = _live(lib, x, mu_law, m.n_classes)
    want = m._epilogue(x[None].astype(np.float64), unbatched_geometry(L), False, WAVE, mu_law)
    assert want.shape == got.shape and np.array_equal(got, want)
    differ = np.flatnonzero(_bits(got) != _bits(want))
    assert np.all(got[differ] == 0), "only the sign of a zero may differ"


def _job(mel=1, T_=26, batched=0, wav=1):
    return cabi.WrnnVocodeJob(mel or None, T_, batched, 2200, 220, 0, 7, wav or None)


def test_live_refusals_without_a_device(lib):
    def refused(job, match, h=None):
        rc = lib.wrnn_vocode_live_start(h, ctypes.byref(job) if job is not None else None, None)
        msg = lib.wrnn_last_error().decode()
        assert rc == cabi.WRNN_E_INVALID and match in msg, (rc, msg)
        return msg
    msg = refused(_job(batched=1), "unbatched")
    assert "last step" in msg
    refused(None, "null job")
    refused(_job(mel=0), "mel and wav are required")
    refused(_job(wav=0), "mel and wav are required")
    refused(_job(T_=20), "T must be >= 21")
    refused(_job(), "null handle")
    n = ctypes.c_int64(-1)
    assert lib.wrnn_vocode_live_poll(None, 0, ctypes.byref(n)) == cabi.WRNN_E_INVALID and n.value == -1
    assert lib.wrnn_debug_live_epilogue(None, 0, WAVE, HOP, 0, 30, None) == cabi.WRNN_E_INVALID
    x, wav = np.zeros(L, np.float32), np.zeros(L)
    assert lib.wrnn_debug_live_epilogue(x.ctypes.data, WAVE + 1, WAVE, HOP, 0, 30, wav.ctypes.data) == cabi.WRNN_E_INVALID


if __name__ == "__main__":
    sys.exit(pytest.main([__file__, "-v", "-s"]))
