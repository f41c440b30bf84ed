"""numpy restatement of librosa 0.6.3's resample(y, orig_sr, target_sr) with its default res_type, resampy's
kaiser_best: resampy.resample (table scaling, interp_delta, output length) and its resample_f loop, then librosa's
fix_length.  Tap by tap, vectorised over outputs, with every step rounded as resampy's arrays round it: float64 weights,
and y kept in the input's dtype (float32) after each tap."""
import numpy as np
import scipy.signal

ZEROS = 64
PRECISION = 16                     # this library's choice (DESIGN.md §3.10); sinc_window's default is 9
BETA = 14.769656459379492
ROLLOFF = 0.9475937167399596


def sinc_window(precision=PRECISION, num_zeros=ZEROS, beta=BETA, rolloff=ROLLOFF):
    """resampy.filters.sinc_window with a Kaiser taper: the float64 half-window of num_zeros * 2^precision + 1 entries."""
    num_bits = 2 ** precision
    n = num_bits * num_zeros
    sinc_win = rolloff * np.sinc(rolloff * np.linspace(0, num_zeros, num=n + 1, endpoint=True))
    taper = scipy.signal.windows.kaiser(2 * n + 1, beta)[n:]
    return taper * sinc_win


_tables = {}


def table(precision=PRECISION):
    if precision not in _tables:
        _tables[precision] = sinc_window(precision)
    return _tables[precision]


def output_length(n, sr_in, sr_out):
    """(resampy's int(n * ratio), librosa's ceil(n * ratio))."""
    ratio = float(sr_out) / sr_in
    return int(n * ratio), int(np.ceil(n * ratio))


def resample(x, sr_in, sr_out, win=None, precision=PRECISION, sequential=False):
    """librosa.resample(x, sr_in, sr_out) for float32 x.  win: the half-window (default: sinc_window(precision)).
    sequential: advance the time register by repeated addition, as resampy does, instead of t * (1 / ratio)."""
    x = np.asarray(x, dtype=np.float32)
    if sr_in == sr_out:
        return x.copy()
    win = table(precision) if win is None else np.asarray(win, dtype=np.float64)
    num_table = 2 ** precision
    ratio = float(sr_out) / sr_in
    n_out, n_len = output_length(x.size, sr_in, sr_out)
    if n_out < 1:
        raise ValueError("no output sample")
    if ratio < 1:
        win = win * ratio
    delta = np.zeros_like(win)
    delta[:-1] = np.diff(win)
    scale = min(1.0, ratio)
    inc = 1.0 / ratio
    step = int(scale * num_table)
    nwin = win.shape[0]
    t = np.arange(n_out)
    if sequential:
        tr = np.concatenate([[0.0], np.cumsum(np.full(n_out - 1, inc))])   # cumsum adds one term at a time
    else:
        tr = t * inc
    n = tr.astype(np.int64)
    frac = scale * (tr - n)
    y = np.zeros(n_out, np.float32)
    xd = x.astype(np.float64)

    def wing(frac, limit, left):
        index_frac = frac * num_table
        offset = index_frac.astype(np.int64)
        eta = index_frac - offset
        taps = np.minimum(limit, (nwin - offset) // step)
        for i in range(int(taps.max(initial=0))):
            m = i < taps
            j = offset[m] + i * step
            weight = win[j] + eta[m] * delta[j]
            src = n[m] - i if left else n[m] + i + 1
            y[m] = (y[m].astype(np.float64) + weight * xd[src]).astype(np.float32)

    wing(frac, n + 1, True)
    wing(scale - frac, x.size - n - 1, False)
    out = np.zeros(n_len, np.float32)
    out[:n_out] = y
    return out
