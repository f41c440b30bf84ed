"""ctypes binding of include/wavernn_b200.h -- the only way the Python host reaches the
CUDA engine.  No torch types cross this boundary: raw pointers (tensor.data_ptr())
and a raw cudaStream_t.  Import never fails (so CPU-only tools can load the package)
but `load()` raises if the shared library has not been built: there is no fallback.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

LIB_NAME = "libwavernn_b200.so"
LIB_PATH = Path(__file__).with_name(LIB_NAME)

WRNN_OK, WRNN_E_INVALID, WRNN_E_CUDA, WRNN_E_NO_DEVICE, WRNN_E_WATCHDOG, WRNN_E_BUSY = 0, -1, -2, -3, -4, -5
MODE_MOL, MODE_RAW = 0, 1
PREC_F16, PREC_FP32, PREC_BF16 = 0, 1, 2
ENGINE_AUTO, ENGINE_SIMT, ENGINE_TCGEN05, ENGINE_STREAM = 0, 1, 2, 3
COND_AUTO, COND_EXPAND, COND_IN_KERNEL = 0, 1, 2
ABI_VERSION = 5

EXPORTS = ("wrnn_abi_version", "wrnn_last_error", "wrnn_create", "wrnn_destroy", "wrnn_generate",
           "wrnn_check", "wrnn_generate_host", "wrnn_engine_name", "wrnn_grid_ctas", "wrnn_launch_count",
           "wrnn_mt19937_uniform", "wrnn_mt19937_uniform_cols", "wrnn_epilogue", "wrnn_expand_conditioning",
           "wrnn_attach_upsampler", "wrnn_conditioning_frames", "wrnn_vocode", "wrnn_vocode_host",
           "wrnn_vocode_many", "wrnn_vocode_many_host", "wrnn_score", "wrnn_score_many", "wrnn_score_many_host",
           "wrnn_vocode_live_start", "wrnn_vocode_live_poll", "wrnn_vocode_many_live_start",
           "wrnn_vocode_many_live_poll", "wrnn_live_open", "wrnn_live_submit", "wrnn_live_cancel", "wrnn_live_poll",
           "wrnn_live_close", "wrnn_mel_create", "wrnn_mel_destroy", "wrnn_melspectrogram_many",
           "wrnn_melspectrogram_many_host", "wrnn_score_wav_many", "wrnn_score_wav_many_host", "wrnn_griffinlim_many",
           "wrnn_griffinlim_many_host", "wrnn_resample_length", "wrnn_resample_many", "wrnn_resample_many_host")
LIVE_RUNNING, LIVE_DONE, LIVE_CANCELLED = 0, 1, 2

_fp = C.POINTER(C.c_float)


class WrnnCfg(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("rnn_dims", "fc_dims", "feat_dims", "aux_dims", "n_classes",
                                         "mode", "precision", "engine")]


WEIGHT_FIELDS = ("I_weight", "I_bias",
                 "rnn1_weight_ih", "rnn1_weight_hh", "rnn1_bias_ih", "rnn1_bias_hh",
                 "rnn2_weight_ih", "rnn2_weight_hh", "rnn2_bias_ih", "rnn2_bias_hh",
                 "fc1_weight", "fc1_bias", "fc2_weight", "fc2_bias", "fc3_weight", "fc3_bias")
# state_dict key for each field (reference models/fatchord_version.py:115-123)
WEIGHT_KEYS = ("I.weight", "I.bias",
               "rnn1.weight_ih_l0", "rnn1.weight_hh_l0", "rnn1.bias_ih_l0", "rnn1.bias_hh_l0",
               "rnn2.weight_ih_l0", "rnn2.weight_hh_l0", "rnn2.bias_ih_l0", "rnn2.bias_hh_l0",
               "fc1.weight", "fc1.bias", "fc2.weight", "fc2.bias", "fc3.weight", "fc3.bias")


class WrnnWeights(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in WEIGHT_FIELDS]


class WrnnJob(C.Structure):
    _fields_ = [("mels_up", C.c_void_p), ("aux", C.c_void_p), ("L", C.c_int64), ("seg_stride", C.c_int64),
                ("n_seg", C.c_int32), ("seg_len", C.c_int32), ("seg_first", C.c_int32), ("steps", C.c_int32),
                ("uniforms", C.c_void_p), ("expo", C.c_void_p),
                ("philox_seed", C.c_uint64), ("philox_offset", C.c_uint64),
                ("out", C.c_void_p), ("x_force", C.c_void_p), ("logits_out", C.c_void_p),
                ("fold_row0", C.c_void_p), ("fold_row_end", C.c_void_p),
                ("mel_frames", C.c_void_p), ("aux_frames", C.c_void_p), ("up_taps", C.c_void_p),
                ("hop", C.c_int32), ("cond_mode", C.c_int32), ("uniforms_ready", C.c_void_p)]


class WrnnTensor(C.Structure):
    _fields_ = [("name", C.c_char_p), ("data", C.c_void_p), ("numel", C.c_int64)]


class WrnnUpsampleCfg(C.Structure):
    _fields_ = [("compute_dims", C.c_int32), ("res_out_dims", C.c_int32), ("res_blocks", C.c_int32), ("pad", C.c_int32),
                ("n_factors", C.c_int32), ("factors", C.c_int32 * 4), ("hop_length", C.c_int32)]


class WrnnVocodeJob(C.Structure):
    _fields_ = [("mel", C.c_void_p), ("T", C.c_int64), ("batched", C.c_int32), ("target", C.c_int32),
                ("overlap", C.c_int32), ("mu_law", C.c_int32), ("philox_seed", C.c_uint64), ("wav", C.c_void_p)]


class WrnnUtterance(C.Structure):
    _fields_ = [("mel", C.c_void_p), ("T", C.c_int64), ("philox_seed", C.c_uint64), ("wav", C.c_void_p)]


class WrnnVocodeBatch(C.Structure):
    _fields_ = [("utts", C.POINTER(WrnnUtterance)), ("n_utts", C.c_int32), ("batched", C.c_int32), ("target", C.c_int32),
                ("overlap", C.c_int32), ("mu_law", C.c_int32)]


class WrnnLiveTicket(C.Structure):
    _fields_ = [("ticket", C.c_int64), ("n_ready", C.c_int64), ("state", C.c_int32), ("pad", C.c_int32)]


class WrnnScoreUtt(C.Structure):
    _fields_ = [("mel", C.c_void_p), ("T", C.c_int64), ("x", C.c_void_p), ("n", C.c_int64), ("nll", C.c_void_p)]


class WrnnMelCfg(C.Structure):
    _fields_ = [("sample_rate", C.c_int32), ("n_fft", C.c_int32), ("hop_length", C.c_int32), ("win_length", C.c_int32),
                ("n_mels", C.c_int32), ("fmin", C.c_float), ("min_level_db", C.c_float)]


class WrnnMelUtt(C.Structure):
    _fields_ = [("y", C.c_void_p), ("n", C.c_int64), ("mel", C.c_void_p)]


class WrnnScoreWavUtt(C.Structure):
    _fields_ = [("y", C.c_void_p), ("n", C.c_int64), ("nll", C.c_void_p)]


class WrnnGlUtt(C.Structure):
    _fields_ = [("mel", C.c_void_p), ("T", C.c_int64), ("phase_seed", C.c_uint64), ("wav", C.c_void_p)]


class WrnnResampleUtt(C.Structure):
    _fields_ = [("x", C.c_void_p), ("n", C.c_int64), ("sample_rate", C.c_int32), ("pad", C.c_int32), ("y", C.c_void_p)]


def resample_utts(utts):
    """A wrnn_resample_utt array over `utts`, a list of (x address, n, sample_rate, y address) (0 = NULL).  Returns the
    array and its length (an empty list gives a NULL array)."""
    arr = (WrnnResampleUtt * max(len(utts), 1))(*[WrnnResampleUtt(x or None, int(n), int(sr), 0, y or None)
                                                  for x, n, sr, y in utts])
    return (arr if utts else None), len(utts)


def mel_cfg(*, sample_rate=22050, n_fft=2048, hop_length=275, win_length=1100, n_mels=80, fmin=40.0,
            min_level_db=-100.0) -> WrnnMelCfg:
    """A wrnn_mel_cfg; the defaults are the reference's hparams."""
    return WrnnMelCfg(int(sample_rate), int(n_fft), int(hop_length), int(win_length), int(n_mels), float(fmin),
                      float(min_level_db))


def ptr_n_ptr_array(struct, items):
    """A wrnn_mel_utt or wrnn_score_wav_utt array over `items`, a list of (address, n, address) (0 = NULL).  Returns
    the array and its length (an empty list gives a NULL array)."""
    arr = (struct * max(len(items), 1))(*[struct(a or None, int(n), b or None) for a, n, b in items])
    return (arr if items else None), len(items)


def gl_utts(utts):
    """A wrnn_gl_utt array over `utts`, a list of (mel address, T, phase_seed, wav address) (0 = NULL).  Returns the
    array and its length (an empty list gives a NULL array)."""
    arr = (WrnnGlUtt * max(len(utts), 1))(*[WrnnGlUtt(m or None, int(T), int(s), w or None) for m, T, s, w in utts])
    return (arr if utts else None), len(utts)


def score_utts(utts):
    """A wrnn_score_utt array over `utts`, a list of (mel address, T, x address, n, nll address) (0 = NULL).  Returns
    the array and its length (an empty list gives a NULL array)."""
    arr = (WrnnScoreUtt * max(len(utts), 1))(*[WrnnScoreUtt(m or None, int(T), x or None, int(n), o or None)
                                               for m, T, x, n, o in utts])
    return (arr if utts else None), len(utts)


def vocode_batch(utts, *, batched=True, target=11000, overlap=550, mu_law=False):
    """A wrnn_vocode_batch over `utts`, a list of (mel address, T, philox_seed, wav address) (0 = NULL).  Returns the
    struct and the utterance array it points to (keep both alive for the call)."""
    arr = (WrnnUtterance * max(len(utts), 1))(*[WrnnUtterance(m or None, int(T), int(s), w or None) for m, T, s, w in utts])
    b = WrnnVocodeBatch(arr if utts else None, len(utts), int(bool(batched)), int(target), int(overlap), int(bool(mu_law)))
    return b, arr


_lib = None


def is_built() -> bool:
    return LIB_PATH.is_file()


def load() -> C.CDLL:
    """dlopen the engine.  Raises RuntimeError if it is missing (no CPU fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    path = os.environ.get("WAVERNN_B200_LIB", str(LIB_PATH))
    if not os.path.isfile(path):
        raise RuntimeError(
            f"wavernn_b200: CUDA engine {path} is not built. Run `python -c 'import __graft_entry__ as g; "
            f"g.build()'` (or `make -C wavernn_b200/csrc`). There is no CPU fallback for generate().")
    lib = C.CDLL(path, mode=C.RTLD_GLOBAL)
    lib.wrnn_abi_version.restype = C.c_int
    lib.wrnn_last_error.restype = C.c_char_p
    lib.wrnn_create.restype = C.c_int
    lib.wrnn_create.argtypes = [C.POINTER(C.c_void_p), C.POINTER(WrnnCfg), C.POINTER(WrnnWeights), C.c_int]
    lib.wrnn_destroy.restype = None
    lib.wrnn_destroy.argtypes = [C.c_void_p]
    lib.wrnn_generate.restype = C.c_int
    lib.wrnn_generate.argtypes = [C.c_void_p, C.POINTER(WrnnJob), C.c_void_p]
    lib.wrnn_check.restype = C.c_int
    lib.wrnn_check.argtypes = [C.c_void_p]
    lib.wrnn_generate_host.restype = C.c_int
    lib.wrnn_generate_host.argtypes = [C.c_void_p, C.POINTER(WrnnJob)]
    lib.wrnn_engine_name.restype = C.c_char_p
    lib.wrnn_engine_name.argtypes = [C.c_void_p]
    lib.wrnn_grid_ctas.restype = C.c_int
    lib.wrnn_grid_ctas.argtypes = [C.c_void_p]
    lib.wrnn_launch_count.restype = C.c_int64
    lib.wrnn_launch_count.argtypes = [C.c_void_p]
    lib.wrnn_expand_conditioning.restype = C.c_int
    lib.wrnn_expand_conditioning.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_int64,
                                             C.c_void_p, C.c_void_p, C.c_void_p]
    lib.wrnn_epilogue.restype = C.c_int
    lib.wrnn_epilogue.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.c_int32, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p]
    lib.wrnn_mt19937_uniform.restype = C.c_int32
    lib.wrnn_mt19937_uniform.argtypes = [C.c_void_p, C.c_int32, C.c_uint64, C.c_void_p, C.c_uint64, C.c_float, C.c_float]
    lib.wrnn_mt19937_uniform_cols.restype = C.c_int32
    lib.wrnn_mt19937_uniform_cols.argtypes = [C.c_void_p, C.c_int32, C.c_uint64, C.c_void_p, C.c_uint64, C.c_uint64,
                                              C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64, C.c_float, C.c_float]
    lib.wrnn_attach_upsampler.restype = C.c_int
    lib.wrnn_attach_upsampler.argtypes = [C.c_void_p, C.POINTER(WrnnUpsampleCfg), C.POINTER(WrnnTensor), C.c_int32]
    lib.wrnn_conditioning_frames.restype = C.c_int
    lib.wrnn_conditioning_frames.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.wrnn_vocode.restype = C.c_int
    lib.wrnn_vocode.argtypes = [C.c_void_p, C.POINTER(WrnnVocodeJob), C.c_void_p]
    lib.wrnn_vocode_host.restype = C.c_int
    lib.wrnn_vocode_host.argtypes = [C.c_void_p, C.POINTER(WrnnVocodeJob)]
    lib.wrnn_vocode_many.restype = C.c_int
    lib.wrnn_vocode_many.argtypes = [C.c_void_p, C.POINTER(WrnnVocodeBatch), C.c_void_p]
    lib.wrnn_vocode_many_host.restype = C.c_int
    lib.wrnn_vocode_many_host.argtypes = [C.c_void_p, C.POINTER(WrnnVocodeBatch)]
    lib.wrnn_score.restype = C.c_int
    lib.wrnn_score.argtypes = [C.c_void_p, C.POINTER(WrnnJob), C.c_void_p, C.c_void_p]
    lib.wrnn_score_many.restype = C.c_int
    lib.wrnn_score_many.argtypes = [C.c_void_p, C.POINTER(WrnnScoreUtt), C.c_int32, C.c_void_p]
    lib.wrnn_score_many_host.restype = C.c_int
    lib.wrnn_score_many_host.argtypes = [C.c_void_p, C.POINTER(WrnnScoreUtt), C.c_int32]
    lib.wrnn_vocode_live_start.restype = C.c_int
    lib.wrnn_vocode_live_start.argtypes = [C.c_void_p, C.POINTER(WrnnVocodeJob), C.c_void_p]
    lib.wrnn_vocode_live_poll.restype = C.c_int
    lib.wrnn_vocode_live_poll.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_int64)]
    lib.wrnn_vocode_many_live_start.restype = C.c_int
    lib.wrnn_vocode_many_live_start.argtypes = [C.c_void_p, C.POINTER(WrnnVocodeBatch), C.c_void_p]
    lib.wrnn_vocode_many_live_poll.restype = C.c_int
    lib.wrnn_vocode_many_live_poll.argtypes = [C.c_void_p, C.c_int32, C.c_void_p]
    lib.wrnn_live_open.restype = C.c_int
    lib.wrnn_live_open.argtypes = [C.c_void_p, C.c_int32, C.c_int64, C.c_int32, C.c_void_p]
    lib.wrnn_live_submit.restype = C.c_int
    lib.wrnn_live_submit.argtypes = [C.c_void_p, C.POINTER(WrnnUtterance), C.POINTER(C.c_int64)]
    lib.wrnn_live_cancel.restype = C.c_int
    lib.wrnn_live_cancel.argtypes = [C.c_void_p, C.c_int64]
    lib.wrnn_live_poll.restype = C.c_int
    lib.wrnn_live_poll.argtypes = [C.c_void_p, C.c_int32, C.POINTER(WrnnLiveTicket), C.c_int32, C.POINTER(C.c_int32)]
    lib.wrnn_live_close.restype = C.c_int
    lib.wrnn_live_close.argtypes = [C.c_void_p]
    lib.wrnn_mel_create.restype = C.c_int
    lib.wrnn_mel_create.argtypes = [C.POINTER(C.c_void_p), C.POINTER(WrnnMelCfg), C.c_int]
    lib.wrnn_mel_destroy.restype = None
    lib.wrnn_mel_destroy.argtypes = [C.c_void_p]
    lib.wrnn_melspectrogram_many.restype = C.c_int
    lib.wrnn_melspectrogram_many.argtypes = [C.c_void_p, C.POINTER(WrnnMelUtt), C.c_int32, C.c_void_p]
    lib.wrnn_melspectrogram_many_host.restype = C.c_int
    lib.wrnn_melspectrogram_many_host.argtypes = [C.c_void_p, C.POINTER(WrnnMelUtt), C.c_int32]
    lib.wrnn_score_wav_many.restype = C.c_int
    lib.wrnn_score_wav_many.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(WrnnScoreWavUtt), C.c_int32, C.c_int32, C.c_int32,
                                        C.c_void_p]
    lib.wrnn_score_wav_many_host.restype = C.c_int
    lib.wrnn_score_wav_many_host.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(WrnnScoreWavUtt), C.c_int32, C.c_int32,
                                             C.c_int32]
    lib.wrnn_resample_length.restype = C.c_int64
    lib.wrnn_resample_length.argtypes = [C.c_int64, C.c_int32, C.c_int32]
    lib.wrnn_resample_many.restype = C.c_int
    lib.wrnn_resample_many.argtypes = [C.c_void_p, C.POINTER(WrnnResampleUtt), C.c_int32, C.c_void_p]
    lib.wrnn_resample_many_host.restype = C.c_int
    lib.wrnn_resample_many_host.argtypes = [C.c_void_p, C.POINTER(WrnnResampleUtt), C.c_int32]
    lib.wrnn_griffinlim_many.restype = C.c_int
    lib.wrnn_griffinlim_many.argtypes = [C.c_void_p, C.POINTER(WrnnGlUtt), C.c_int32, C.c_int32, C.c_void_p]
    lib.wrnn_griffinlim_many_host.restype = C.c_int
    lib.wrnn_griffinlim_many_host.argtypes = [C.c_void_p, C.POINTER(WrnnGlUtt), C.c_int32, C.c_int32]
    # test hooks (not declared in the header)
    lib.wrnn_debug_resample_table.restype = C.c_int64
    lib.wrnn_debug_resample_table.argtypes = [C.c_void_p]
    lib.wrnn_debug_resample.restype = C.c_int
    lib.wrnn_debug_resample.argtypes = [C.POINTER(WrnnResampleUtt), C.c_int32, C.c_int32]
    lib.wrnn_debug_griffinlim_plan.restype = C.c_int
    lib.wrnn_debug_griffinlim_plan.argtypes = [C.POINTER(WrnnMelCfg), C.POINTER(WrnnGlUtt), C.c_int32, C.c_int32, C.c_void_p]
    lib.wrnn_debug_griffinlim.restype = C.c_int
    lib.wrnn_debug_griffinlim.argtypes = [C.POINTER(WrnnMelCfg), C.c_void_p, C.c_int64, C.c_uint64, C.c_int32, C.c_void_p,
                                          C.c_void_p]
    lib.wrnn_debug_mel_tables.restype = C.c_int
    lib.wrnn_debug_mel_tables.argtypes = [C.POINTER(WrnnMelCfg), C.c_void_p, C.c_void_p, C.c_void_p]
    lib.wrnn_debug_mel_plan.restype = C.c_int
    lib.wrnn_debug_mel_plan.argtypes = [C.POINTER(WrnnMelCfg), C.POINTER(WrnnMelUtt), C.c_int32, C.c_void_p]
    lib.wrnn_debug_mel_frames.restype = C.c_int
    lib.wrnn_debug_mel_frames.argtypes = [C.POINTER(WrnnMelCfg), C.c_void_p, C.c_int64, C.c_void_p]
    lib.wrnn_debug_score_wav_plan.restype = C.c_int
    lib.wrnn_debug_score_wav_plan.argtypes = [C.c_int32, C.c_int32, C.POINTER(WrnnMelCfg), C.POINTER(WrnnScoreWavUtt),
                                              C.c_int32, C.c_void_p]
    lib.wrnn_debug_wav_targets.restype = C.c_int
    lib.wrnn_debug_wav_targets.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]
    lib.wrnn_debug_score_wav_targets.restype = C.c_int
    lib.wrnn_debug_score_wav_targets.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                                 C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.wrnn_debug_live_session_deliver.restype = C.c_int
    lib.wrnn_debug_live_session_deliver.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p,
                                                    C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.wrnn_debug_live_tag.restype = C.c_uint32
    lib.wrnn_debug_live_tag.argtypes = [C.c_int64]
    lib.wrnn_debug_live_session_slot.restype = C.c_int
    lib.wrnn_debug_live_session_slot.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.c_int32, C.c_uint32, C.c_uint32,
                                                 C.c_uint64, C.c_int64, C.c_void_p]
    lib.wrnn_debug_live_many_deliver.restype = C.c_int
    lib.wrnn_debug_live_many_deliver.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32,
                                                 C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
    lib.wrnn_debug_live_epilogue.restype = C.c_int
    lib.wrnn_debug_live_epilogue.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]
    lib.wrnn_debug_score_many_plan.restype = C.c_int
    lib.wrnn_debug_score_many_plan.argtypes = [C.c_int32, C.POINTER(WrnnScoreUtt), C.c_int32, C.c_void_p, C.c_void_p]
    lib.wrnn_debug_vocode_many_plan.restype = C.c_int
    lib.wrnn_debug_vocode_many_plan.argtypes = [C.c_int32, C.POINTER(WrnnVocodeBatch), C.c_void_p, C.c_void_p, C.c_void_p]
    lib.wrnn_debug_fold_geometry.restype = C.c_int
    lib.wrnn_debug_fold_geometry.argtypes = [C.c_int64, C.c_int32, C.c_int64, C.c_int64, C.c_void_p]
    lib.wrnn_debug_epilogue_tables.restype = C.c_int
    lib.wrnn_debug_epilogue_tables.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                               C.c_void_p, C.c_void_p]
    lib.wrnn_debug_upsampler.restype = C.c_int
    lib.wrnn_debug_upsampler.argtypes = [C.POINTER(WrnnUpsampleCfg), C.POINTER(WrnnTensor), C.c_int32, C.c_void_p,
                                         C.POINTER(C.c_uint64), C.c_void_p]
    if lib.wrnn_abi_version() != ABI_VERSION:
        raise RuntimeError(f"wavernn_b200: ABI mismatch (lib {lib.wrnn_abi_version()} != binding {ABI_VERSION})")
    _lib = lib
    return lib


class EngineError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"wavernn_b200 engine error {code}: {msg}")
        self.code = code


def _check(lib, rc: int):
    if rc != 0:
        raise EngineError(rc, (lib.wrnn_last_error() or b"").decode(errors="replace"))


class Engine:
    """Owns one `wrnn_t*`.  `weights` maps WEIGHT_KEYS -> object with .data_ptr()
    (torch tensors, fp32, contiguous, host or device) or raw ints."""

    def __init__(self, weights: dict, *, rnn_dims=512, fc_dims=512, feat_dims=80, aux_dims=32, n_classes=30,
                 mode="MOL", precision="fp16", engine="auto", device: int = 0):
        self._h = C.c_void_p()
        self.lib = load()
        cfg = WrnnCfg(rnn_dims, fc_dims, feat_dims, aux_dims, n_classes,
                      {"MOL": MODE_MOL, "RAW": MODE_RAW}[mode],
                      {"fp16": PREC_F16, "bf16": PREC_BF16, "fp32": PREC_FP32}[precision],
                      {"auto": ENGINE_AUTO, "simt": ENGINE_SIMT, "tcgen05": ENGINE_TCGEN05, "stream": ENGINE_STREAM}[engine])
        w = WrnnWeights()
        keep = []
        for field, key in zip(WEIGHT_FIELDS, WEIGHT_KEYS):
            t = weights[key]
            if hasattr(t, "data_ptr"):
                t = t.detach()
                if t.dtype is not _torch().float32 or not t.is_contiguous():
                    t = t.float().contiguous()
                keep.append(t)
                setattr(w, field, t.data_ptr())
            else:
                setattr(w, field, int(t))
        _check(self.lib, self.lib.wrnn_create(C.byref(self._h), C.byref(cfg), C.byref(w), int(device)))
        del keep
        self.n_classes, self.mode, self.precision, self.device = n_classes, mode, precision, device

    @property
    def name(self) -> str:
        return self.lib.wrnn_engine_name(self._h).decode()

    @property
    def grid_ctas(self) -> int:
        return self.lib.wrnn_grid_ctas(self._h)

    @property
    def launch_count(self) -> int:
        return self.lib.wrnn_launch_count(self._h)

    def generate(self, *, mels_up: int, aux: int, L: int, n_seg: int, seg_len: int, seg_stride: int, out: int,
                 seg_first: int = 0, steps: int = 0, uniforms: int = 0, expo: int = 0, philox_seed: int = 0,
                 philox_offset: int = 0, x_force: int = 0, logits_out: int = 0, fold_row0: int = 0, fold_row_end: int = 0,
                 mel_frames: int = 0, aux_frames: int = 0, up_taps: int = 0, hop: int = 0, cond_mode: int = 0,
                 uniforms_ready: int = 0, stream: int = 0):
        """All buffer arguments are raw device addresses (ints).  Asynchronous."""
        job = WrnnJob(mels_up, aux, L, seg_stride, n_seg, seg_len, seg_first, steps, uniforms or None,
                      expo or None, philox_seed, philox_offset, out, x_force or None, logits_out or None,
                      fold_row0 or None, fold_row_end or None, mel_frames or None, aux_frames or None, up_taps or None,
                      hop, cond_mode, uniforms_ready or None)
        _check(self.lib, self.lib.wrnn_generate(self._h, C.byref(job), C.c_void_p(stream or None)))

    def generate_host(self, *, mels_up, aux, n_seg: int, seg_len: int, seg_stride: int, seg_first: int = 0, steps: int = 0,
                      uniforms=None, expo=None, philox_seed: int = 0, philox_offset: int = 0, x_force=None,
                      want_logits: bool = False):
        """wrnn_generate_host: the same job with HOST buffers (numpy float32 arrays) -- the entry a non-torch caller
        binds.  Copies in, runs, copies out, synchronises and checks.  Returns samples (n_seg, S)[, logits (S, n_seg, C)]."""
        import numpy as np
        f32 = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.float32)
        mels_up, aux, uniforms, expo, x_force = f32(mels_up), f32(aux), f32(uniforms), f32(expo), f32(x_force)
        S = steps or seg_len
        out = np.empty((n_seg, S), dtype=np.float32)
        logits = np.empty((S, n_seg, self.n_classes), dtype=np.float32) if want_logits else None
        ptr = lambda a: None if a is None else a.ctypes.data
        job = WrnnJob(ptr(mels_up), ptr(aux), mels_up.shape[0], seg_stride, n_seg, seg_len, seg_first, steps, ptr(uniforms),
                      ptr(expo), philox_seed, philox_offset, ptr(out), ptr(x_force), ptr(logits), None, None, None, None,
                      None, 0, 0, None)
        _check(self.lib, self.lib.wrnn_generate_host(self._h, C.byref(job)))
        return (out, logits) if want_logits else out

    # ---- from a mel, through the library alone (wrnn_attach_upsampler / wrnn_vocode) ----
    def attach_upsampler(self, state_dict: dict, *, compute_dims=128, res_out_dims=128, res_blocks=10, pad=2,
                         upsample_factors=(5, 5, 11), hop_length=275):
        """wrnn_attach_upsampler with the `upsample.*` entries of `state_dict` (torch tensors on any device, or numpy
        arrays); the WaveRNN ctor arguments of the same names describe the network."""
        cfg = upsample_cfg(compute_dims=compute_dims, res_out_dims=res_out_dims, res_blocks=res_blocks, pad=pad,
                           upsample_factors=upsample_factors, hop_length=hop_length)
        arr, keep = tensor_list(state_dict)
        _check(self.lib, self.lib.wrnn_attach_upsampler(self._h, C.byref(cfg), arr, len(arr)))
        del keep
        self.hop_length = int(hop_length)

    def conditioning_frames(self, *, mel: int, T: int, mel_frames: int, aux_frames: int, up_taps: int = 0, stream: int = 0):
        """wrnn_conditioning_frames with raw device addresses: mel [80, T] -> mel_frames [T+4, 80], aux_frames [T, 128]
        (and up_taps [hop, 5] unless 0).  Asynchronous on `stream`."""
        _check(self.lib, self.lib.wrnn_conditioning_frames(self._h, mel, int(T), mel_frames, aux_frames, up_taps or None,
                                                           stream or None))

    def vocode(self, *, mel: int, T: int, wav: int, batched: bool = True, target: int = 11000, overlap: int = 550,
               mu_law: bool = False, philox_seed: int = 0, stream: int = 0):
        """wrnn_vocode with raw device addresses: mel [80, T] fp32 -> wav [(T-1)*hop] float64.  Asynchronous."""
        job = WrnnVocodeJob(mel, int(T), int(bool(batched)), int(target), int(overlap), int(bool(mu_law)), int(philox_seed), wav)
        _check(self.lib, self.lib.wrnn_vocode(self._h, C.byref(job), C.c_void_p(stream or None)))

    def vocode_host(self, mel, *, batched: bool = True, target: int = 11000, overlap: int = 550, mu_law: bool = False,
                    philox_seed: int = 0):
        """wrnn_vocode_host: mel (80, T) numpy -> float64 waveform of (T-1)*hop samples, what generate(mel[None], None,
        batched, target, overlap, mu_law) returns with gen_rng='philox' -- without torch."""
        mel, wav = self._mel_and_wav(mel)
        job = WrnnVocodeJob(mel.ctypes.data, mel.shape[-1], int(bool(batched)), int(target), int(overlap), int(bool(mu_law)),
                            int(philox_seed), wav.ctypes.data)
        _check(self.lib, self.lib.wrnn_vocode_host(self._h, C.byref(job)))
        return wav

    def vocode_many(self, *, mels, Ts, seeds, wavs, batched: bool = True, target: int = 11000, overlap: int = 550,
                    mu_law: bool = False, stream: int = 0):
        """wrnn_vocode_many with raw device addresses: utterance i is mels[i] [80, Ts[i]] fp32 -> wavs[i]
        [(Ts[i]-1)*hop] float64, keyed by seeds[i].  One job for the whole batch.  Asynchronous."""
        b, keep = vocode_batch(list(zip(mels, Ts, seeds, wavs)), batched=batched, target=target, overlap=overlap,
                               mu_law=mu_law)
        _check(self.lib, self.lib.wrnn_vocode_many(self._h, C.byref(b), C.c_void_p(stream or None)))
        del keep

    def vocode_many_host(self, mels, seeds, *, batched: bool = True, target: int = 11000, overlap: int = 550,
                         mu_law: bool = False):
        """wrnn_vocode_many_host: a list of numpy mels (80, T_i) and one Philox seed per mel -> the list of float64
        waveforms, each bit-identical to vocode_host(mel_i, philox_seed=seeds[i]) on a handle with a fixed engine."""
        pairs = [self._mel_and_wav(m) for m in mels]
        mels, wavs = [m for m, _ in pairs], [w for _, w in pairs]
        if len(seeds) != len(mels):
            raise ValueError("one seed per mel")
        b, keep = vocode_batch([(m.ctypes.data, m.shape[-1], s, w.ctypes.data) for m, s, w in zip(mels, seeds, wavs)],
                               batched=batched, target=target, overlap=overlap, mu_law=mu_law)
        _check(self.lib, self.lib.wrnn_vocode_many_host(self._h, C.byref(b)))
        del keep
        return wavs

    def vocode_live(self, mel, *, philox_seed: int, mu_law: bool = False, wait_us: int = 1000):
        """wrnn_vocode_live_start / _poll: a generator over the float64 waveform of the unbatched vocode_host(mel,
        batched=False, mu_law=mu_law, philox_seed=philox_seed), yielding each newly final slice while the kernel is still
        generating (views of one array; their concatenation is bit-identical to vocode_host's).  Each poll waits up to
        wait_us.  Closing the generator early still waits for the job, which cannot be cancelled."""
        mel, wav = self._mel_and_wav(mel)
        job = WrnnVocodeJob(mel.ctypes.data, mel.shape[-1], 0, 0, 0, int(bool(mu_law)), int(philox_seed), wav.ctypes.data)
        _check(self.lib, self.lib.wrnn_vocode_live_start(self._h, C.byref(job), None))
        n, prev, rc = C.c_int64(0), 0, 1
        try:
            while rc == 1:
                rc = self.lib.wrnn_vocode_live_poll(self._h, int(wait_us), C.byref(n))
                if rc < 0:
                    _check(self.lib, rc)
                if n.value > prev:
                    yield wav[prev:n.value]
                    prev = n.value
        finally:
            while rc == 1:                               # closed early: the job runs to its end, into `wav`
                rc = self.lib.wrnn_vocode_live_poll(self._h, 100000, C.byref(n))

    def vocode_many_live(self, mels, seeds, *, mu_law: bool = False, wait_us: int = 1000):
        """wrnn_vocode_many_live_start / _poll: a generator over the float64 waveforms of the unbatched
        vocode_many_host(mels, seeds, batched=False, mu_law=mu_law) (up to 64 mels), yielding (i, slice) for each newly
        final slice of waveform i while the kernel is still generating (views of one array per mel; the concatenation
        of utterance i's slices is bit-identical to vocode_many_host's waveform i).  Each poll waits up to wait_us.
        Closing the generator early still waits for the job, which cannot be cancelled."""
        import numpy as np
        pairs = [self._mel_and_wav(m) for m in mels]
        mels, wavs = [m for m, _ in pairs], [w for _, w in pairs]
        if len(seeds) != len(mels):
            raise ValueError("one seed per mel")
        b, keep = vocode_batch([(m.ctypes.data, m.shape[-1], s, w.ctypes.data) for m, s, w in zip(mels, seeds, wavs)],
                               batched=False, mu_law=mu_law)
        _check(self.lib, self.lib.wrnn_vocode_many_live_start(self._h, C.byref(b), None))
        del keep
        n = np.zeros(len(mels), dtype=np.int64)
        prev, rc = n.copy(), 1
        try:
            while rc == 1:
                rc = self.lib.wrnn_vocode_many_live_poll(self._h, int(wait_us), n.ctypes.data)
                if rc < 0:
                    _check(self.lib, rc)
                for i in np.flatnonzero(n > prev):
                    yield int(i), wavs[i][prev[i]:n[i]]
                    prev[i] = n[i]
        finally:
            while rc == 1:                               # closed early: the job runs to its end, into `wavs`
                rc = self.lib.wrnn_vocode_many_live_poll(self._h, 100000, n.ctypes.data)

    def _mel_and_wav(self, mel):
        """mel (80, T) or (1, 80, T) as a contiguous float32 (80, T) array, and a zeroed float64 waveform of its
        (T - 1) * hop samples."""
        import numpy as np
        mel = np.ascontiguousarray(mel, dtype=np.float32)
        if mel.ndim == 3 and mel.shape[0] == 1:
            mel = mel[0]
        return mel, np.zeros(max(mel.shape[-1] - 1, 0) * getattr(self, "hop_length", 275), dtype=np.float64)

    def live_session(self, capacity: int, max_T: int, mu_law: bool = False):
        """wrnn_live_open: a LiveSession of `capacity` slots (1 to 64) for mels of up to max_T frames, into whose running
        kernel each submitted mel is admitted at the next boundary.  Use it as a context manager (close on exit)."""
        return LiveSession(self, capacity, max_T, mu_law)

    # ---- scoring (wrnn_score / wrnn_score_many): the reference's training loss per sample, teacher-forced ----
    def score(self, *, L: int, n_seg: int, seg_len: int, seg_stride: int, x_force: int, nll: int, mels_up: int = 0, aux: int = 0,
              seg_first: int = 0, steps: int = 0, logits_out: int = 0, fold_row0: int = 0, fold_row_end: int = 0,
              mel_frames: int = 0, aux_frames: int = 0, up_taps: int = 0, hop: int = 0, cond_mode: int = 0, stream: int = 0):
        """wrnn_score with raw device addresses: nll [seg_len, n_seg] fp32 = the loss of target x_force[t] (same layout)
        given x_force[:t] and the conditioning rows up to t.  The job is wrnn_generate's without `out` or draws.
        Asynchronous."""
        job = WrnnJob(mels_up or None, aux or None, L, seg_stride, n_seg, seg_len, seg_first, steps, None, None, 0, 0, None,
                      x_force or None, logits_out or None, fold_row0 or None, fold_row_end or None, mel_frames or None,
                      aux_frames or None, up_taps or None, hop, cond_mode, None)
        _check(self.lib, self.lib.wrnn_score(self._h, C.byref(job), nll or None, C.c_void_p(stream or None)))

    def score_many(self, *, mels, Ts, xs, ns, nlls, stream: int = 0):
        """wrnn_score_many with raw device addresses: utterance i is mels[i] [80, Ts[i]] and its waveform xs[i] [ns[i]]
        -> nlls[i] [ns[i]] fp32, each scored unbatched (one fold).  One job for the whole batch.  Asynchronous."""
        arr, n = score_utts(list(zip(mels, Ts, xs, ns, nlls)))
        _check(self.lib, self.lib.wrnn_score_many(self._h, arr, n, C.c_void_p(stream or None)))

    def score_many_host(self, mels, xs):
        """wrnn_score_many_host: a list of numpy mels (80, T_i) and the waveforms xs[i] (n_i samples, n_i <= T_i * hop)
        -> the list of per-sample losses (nats, float32), without torch."""
        import numpy as np
        mels = [self._mel_and_wav(m)[0] for m in mels]
        xs = [np.ascontiguousarray(x, dtype=np.float32).reshape(-1) for x in xs]
        if len(xs) != len(mels):
            raise ValueError("one waveform per mel")
        nlls = [np.empty(x.size, dtype=np.float32) for x in xs]
        arr, n = score_utts([(m.ctypes.data, m.shape[-1], x.ctypes.data, x.size, o.ctypes.data)
                             for m, x, o in zip(mels, xs, nlls)])
        _check(self.lib, self.lib.wrnn_score_many_host(self._h, arr, n))
        return nlls

    def score_wav_many(self, analysis: "MelAnalysis", *, ys, ns, nlls, peak_norm: bool = False, mu_law: bool = False,
                       stream: int = 0):
        """wrnn_score_wav_many with raw device addresses: recording i is ys[i] [ns[i]] fp32 -> nlls[i] [ns[i]], its mel
        made by `analysis` and its targets quantised as preprocess.py stores them.  Asynchronous."""
        arr, n = ptr_n_ptr_array(WrnnScoreWavUtt, list(zip(ys, ns, nlls)))
        _check(self.lib, self.lib.wrnn_score_wav_many(self._h, analysis._m, arr, n, int(bool(peak_norm)), int(bool(mu_law)),
                                                      C.c_void_p(stream or None)))

    def score_wav_many_host(self, analysis: "MelAnalysis", ys, *, peak_norm: bool = False, mu_law: bool = False):
        """wrnn_score_wav_many_host: a list of numpy recordings (float32) -> the list of per-sample losses (nats,
        float32): the loss train_wavernn.py would report on each recording, from its audio alone."""
        import numpy as np
        ys = [np.ascontiguousarray(y, dtype=np.float32).reshape(-1) for y in ys]
        nlls = [np.empty(y.size, dtype=np.float32) for y in ys]
        arr, n = ptr_n_ptr_array(WrnnScoreWavUtt, [(y.ctypes.data, y.size, o.ctypes.data) for y, o in zip(ys, nlls)])
        _check(self.lib, self.lib.wrnn_score_wav_many_host(self._h, analysis._m, arr, n, int(bool(peak_norm)),
                                                           int(bool(mu_law))))
        return nlls

    def check(self):
        _check(self.lib, self.lib.wrnn_check(self._h))

    def close(self):
        if self._h:
            self.lib.wrnn_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class MelAnalysis:
    """Owns one `wrnn_mel_t*`: the reference's melspectrogram(y) on the device, for the wrnn_mel_cfg built from the
    keyword arguments (cabi.mel_cfg; defaults are the reference's hparams)."""

    def __init__(self, *, device: int = 0, **cfg):
        self._m = C.c_void_p()
        self.lib = load()
        self.cfg = mel_cfg(**cfg)
        _check(self.lib, self.lib.wrnn_mel_create(C.byref(self._m), C.byref(self.cfg), int(device)))

    def frames(self, n: int) -> int:
        """Frames of the mel of n samples: 1 + n // hop_length."""
        return 1 + int(n) // self.cfg.hop_length

    def melspectrogram_many(self, *, ys, ns, mels, stream: int = 0):
        """wrnn_melspectrogram_many with raw device addresses: ys[i] [ns[i]] fp32 -> mels[i] [n_mels, frames(ns[i])].
        Asynchronous."""
        arr, n = ptr_n_ptr_array(WrnnMelUtt, list(zip(ys, ns, mels)))
        _check(self.lib, self.lib.wrnn_melspectrogram_many(self._m, arr, n, C.c_void_p(stream or None)))

    def melspectrogram_many_host(self, ys):
        """wrnn_melspectrogram_many_host: a list of numpy waveforms -> the list of float32 mels [n_mels, T_i]."""
        import numpy as np
        ys = [np.ascontiguousarray(y, dtype=np.float32).reshape(-1) for y in ys]
        mels = [np.empty((self.cfg.n_mels, self.frames(y.size)), dtype=np.float32) for y in ys]
        arr, n = ptr_n_ptr_array(WrnnMelUtt, [(y.ctypes.data, y.size, m.ctypes.data) for y, m in zip(ys, mels)])
        _check(self.lib, self.lib.wrnn_melspectrogram_many_host(self._m, arr, n))
        return mels

    def samples(self, T: int) -> int:
        """Samples of the Griffin-Lim reconstruction of T frames: hop_length * (T - 1)."""
        return self.cfg.hop_length * (int(T) - 1)

    def griffinlim_many(self, *, mels, Ts, seeds, wavs, n_iter: int = 32, stream: int = 0):
        """wrnn_griffinlim_many with raw device addresses: mels[i] [n_mels, Ts[i]] fp32 -> wavs[i] [samples(Ts[i])]
        fp32, the initial phases keyed by seeds[i].  Asynchronous."""
        arr, n = gl_utts(list(zip(mels, Ts, seeds, wavs)))
        _check(self.lib, self.lib.wrnn_griffinlim_many(self._m, arr, n, int(n_iter), C.c_void_p(stream or None)))

    def griffinlim_many_host(self, mels, n_iter: int = 32, seeds=None):
        """wrnn_griffinlim_many_host: a list of numpy mels [n_mels, T_i] and one phase seed per mel (default i) -> the
        list of float32 waveforms [hop_length * (T_i - 1)]."""
        import numpy as np
        mels = [np.ascontiguousarray(m, dtype=np.float32) for m in mels]
        seeds = list(range(len(mels))) if seeds is None else list(seeds)
        if len(seeds) != len(mels):
            raise ValueError("one seed per mel")
        wavs = [np.empty(max(self.samples(m.shape[-1]), 0), dtype=np.float32) for m in mels]
        arr, n = gl_utts([(m.ctypes.data, m.shape[-1], s, w.ctypes.data) for m, s, w in zip(mels, seeds, wavs)])
        _check(self.lib, self.lib.wrnn_griffinlim_many_host(self._m, arr, n, int(n_iter)))
        return wavs

    def resample_length(self, n: int, sample_rate: int) -> int:
        """Samples of a recording of n samples at sample_rate resampled to this object's rate (wrnn_resample_length):
        ceil(n * ratio), what librosa.load returns."""
        return int(self.lib.wrnn_resample_length(int(n), int(sample_rate), self.cfg.sample_rate))

    def resample_many(self, *, xs, ns, rates, ys, stream: int = 0):
        """wrnn_resample_many with raw device addresses: xs[i] [ns[i]] fp32 at rates[i] Hz -> ys[i]
        [resample_length(ns[i], rates[i])] at this object's sample_rate.  Asynchronous."""
        arr, n = resample_utts(list(zip(xs, ns, rates, ys)))
        _check(self.lib, self.lib.wrnn_resample_many(self._m, arr, n, C.c_void_p(stream or None)))

    def resample_many_host(self, xs, rates):
        """wrnn_resample_many_host: a list of numpy recordings and their sample rates -> the list of float32 recordings
        at this object's sample_rate, what librosa.load(..., sr=sample_rate) makes of them after decoding."""
        import numpy as np
        xs = [np.ascontiguousarray(x, dtype=np.float32).reshape(-1) for x in xs]
        rates = [int(r) for r in rates]
        if len(rates) != len(xs):
            raise ValueError("one sample rate per recording")
        ys = [np.empty(max(self.resample_length(x.size, r), 0), dtype=np.float32) for x, r in zip(xs, rates)]
        arr, n = resample_utts([(x.ctypes.data, x.size, r, y.ctypes.data) for x, r, y in zip(xs, rates, ys)])
        _check(self.lib, self.lib.wrnn_resample_many_host(self._m, arr, n))
        return ys

    def close(self):
        if self._m:
            self.lib.wrnn_mel_destroy(self._m)
            self._m = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class LiveSession:
    """wrnn_live_*: submit(mel, philox_seed) -> ticket at any time; poll() yields (ticket, slice) for each newly final
    slice of a ticket's float64 waveform (views of one array per ticket; their concatenation is bit-identical to
    vocode_host(mel, batched=False, mu_law=mu_law, philox_seed=philox_seed)); cancel(ticket); close().  `waves` maps
    each ticket to its array, `states` to its last reported state (LIVE_*)."""

    def __init__(self, engine: Engine, capacity: int, max_T: int, mu_law: bool = False):
        self.engine, self.lib, self.capacity = engine, engine.lib, int(capacity)
        _check(self.lib, self.lib.wrnn_live_open(engine._h, self.capacity, int(max_T), int(bool(mu_law)), None))
        self.open = True
        self.waves, self.states, self._mels, self._prev = {}, {}, {}, {}
        self._out = (WrnnLiveTicket * (2 * self.capacity))()

    def submit(self, mel, *, philox_seed: int) -> int:
        """Submits mel (80, T) numpy; returns its ticket.  Raises EngineError(WRNN_E_BUSY) when every slot is held."""
        mel, wav = self.engine._mel_and_wav(mel)
        u = WrnnUtterance(mel.ctypes.data, mel.shape[-1], int(philox_seed), wav.ctypes.data)
        tk = C.c_int64(0)
        _check(self.lib, self.lib.wrnn_live_submit(self.engine._h, C.byref(u), C.byref(tk)))
        t = int(tk.value)
        self.waves[t], self._mels[t], self._prev[t], self.states[t] = wav, mel, 0, LIVE_RUNNING
        return t

    def cancel(self, ticket: int):
        _check(self.lib, self.lib.wrnn_live_cancel(self.engine._h, int(ticket)))

    def poll_once(self, wait_us: int = 1000):
        """One wrnn_live_poll: returns (rc, [(ticket, slice), ...]) for the slices that became final."""
        n = C.c_int32(0)
        rc = self.lib.wrnn_live_poll(self.engine._h, int(wait_us), self._out, len(self._out), C.byref(n))
        if rc < 0:
            _check(self.lib, rc)
        got = []
        for e in self._out[:n.value]:
            t = int(e.ticket)
            if int(e.n_ready) > self._prev[t]:
                got.append((t, self.waves[t][self._prev[t]:int(e.n_ready)]))
                self._prev[t] = int(e.n_ready)
            self.states[t] = int(e.state)
            if e.state != LIVE_RUNNING:
                self._mels.pop(t, None)
        return rc, got

    def poll(self, wait_us: int = 1000):
        """A generator of (ticket, slice) until no ticket is held."""
        rc = 1
        while rc == 1:
            rc, got = self.poll_once(wait_us)
            yield from got

    def close(self):
        if self.open:
            self.open = False
            _check(self.lib, self.lib.wrnn_live_close(self.engine._h))

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


def _torch():
    import torch
    return torch


def upsample_cfg(*, compute_dims=128, res_out_dims=128, res_blocks=10, pad=2, upsample_factors=(5, 5, 11),
                 hop_length=275) -> WrnnUpsampleCfg:
    f = tuple(int(x) for x in upsample_factors)
    if not 1 <= len(f) <= 4:
        raise ValueError("the C ABI takes 1 to 4 upsample factors")
    return WrnnUpsampleCfg(compute_dims, res_out_dims, res_blocks, pad, len(f), (C.c_int32 * 4)(*(f + (0,) * (4 - len(f)))),
                           hop_length)


def tensor_list(state_dict: dict):
    """The `upsample.*` entries of a state_dict as a wrnn_tensor array (fp32, contiguous; torch tensors keep their
    device, numpy arrays are host memory).  Returns (array, objects to keep alive for the call)."""
    import numpy as np
    keep, items = [], []
    for k, v in state_dict.items():
        if not k.startswith("upsample."):
            continue
        if hasattr(v, "data_ptr"):
            v = v.detach().float().contiguous()
            ptr, n = v.data_ptr(), v.numel()
        else:
            v = np.ascontiguousarray(v, dtype=np.float32)
            ptr, n = v.ctypes.data, v.size
        name = k.encode()
        keep += [v, name]
        items.append((name, ptr, n))
    arr = (WrnnTensor * max(len(items), 1))()
    for i, (name, ptr, n) in enumerate(items):
        arr[i] = WrnnTensor(name, ptr, n)
    return (arr if items else (WrnnTensor * 0)()), keep


def expand_conditioning(*, mel_frames: int, aux_frames: int, up_taps: int, hop: int, row_lo: int, n_rows: int,
                        mels_up: int, aux: int, stream: int = 0):
    """wrnn_expand_conditioning with raw device addresses.  Asynchronous on `stream`."""
    lib = load()
    _check(lib, lib.wrnn_expand_conditioning(mel_frames, aux_frames, up_taps, hop, row_lo, n_rows, mels_up, aux, stream or None))


def epilogue(*, samples: int, n_seg: int, seg_len: int, seg_stride: int, overlap: int, fade_in: int, fade_out: int,
             mu_table: int, n_classes: int, tail: int, tail_len: int, wave_len: int, wav: int, stream: int = 0):
    """wrnn_epilogue with raw device addresses (ints; 0 = NULL).  Asynchronous on `stream`."""
    lib = load()
    _check(lib, lib.wrnn_epilogue(samples, n_seg, seg_len, seg_stride, overlap, fade_in or None, fade_out or None,
                                  mu_table or None, n_classes, tail or None, tail_len, wave_len, wav, stream or None))


# ---------------------------------------------------------------------------------------------
# torch CPU generator replay (parity mode's host-side cost; see csrc/wrnn_hostrng.cu)
# ---------------------------------------------------------------------------------------------
# Layout of torch.get_rng_state() for the CPU generator (CPUGeneratorImplStateLegacy): seed u64 @0, left i32 @8,
# seeded i32 @12, next u64 @16, 624 state words as u64 @24, then the cached-normal fields (untouched here).
_MT_N, _MT_OFF, _STATE_BYTES = 624, 24, 5056


def torch_rng_uniform(skip: int, n: int, lo: float, hi: float, out=None, generator=None, row_len: int = 0, cols=None):
    """Advance torch's CPU generator by `skip` discarded 32-bit outputs and then fill `out` (a contiguous CPU float32
    tensor with n elements, e.g. pinned) with what `torch.empty(n).uniform_(lo, hi)` would have produced -- natively.
    The generator (default: the global one) is left in exactly the state torch would have left it in.
    With `row_len` and `cols=((a_lo, a_hi), (b_lo, b_hi))` the n draws are read as an (n // row_len, row_len) matrix of
    which only those two column ranges are kept (`out`: rows x (a_hi-a_lo + b_hi-b_lo)); the rest is skipped unconverted."""
    import numpy as np
    import torch
    lib = load()
    st = (generator.get_state() if generator is not None else torch.get_rng_state()).clone()
    a = st.numpy()
    if a.size != _STATE_BYTES:
        raise RuntimeError("unexpected torch CPU generator state size")
    left = int(a[8:12].view(np.int32)[0])
    if not (1 <= left <= _MT_N):
        raise RuntimeError("unexpected torch CPU generator state (left)")
    words = a[_MT_OFF:_MT_OFF + 8 * _MT_N].view(np.uint64)
    mt = np.ascontiguousarray(words.astype(np.uint32))
    if cols is not None:
        (a_lo, a_hi), (b_lo, b_hi) = cols
        rows = n // row_len
        assert row_len > 0 and rows * row_len == n
        n_out = rows * ((a_hi - a_lo) + (b_hi - b_lo))
    else:
        n_out = n
    if out is None:
        out = torch.empty(n_out, dtype=torch.float32)
    assert out.dtype == torch.float32 and out.is_contiguous() and out.numel() >= n_out and out.device.type == 'cpu'
    if cols is not None:
        pos = lib.wrnn_mt19937_uniform_cols(mt.ctypes.data, _MT_N + 1 - left, int(skip), out.data_ptr(), rows, int(row_len),
                                            int(a_lo), int(a_hi), int(b_lo), int(b_hi), float(lo), float(hi))
    else:
        pos = lib.wrnn_mt19937_uniform(mt.ctypes.data, _MT_N + 1 - left, int(skip), out.data_ptr() if n else None, int(n),
                                       float(lo), float(hi))
    if pos < 0:
        raise RuntimeError("wrnn_mt19937_uniform rejected its arguments")
    words[:] = mt
    a[8:12].view(np.int32)[0] = _MT_N + 1 - pos
    a[16:24].view(np.uint64)[0] = pos
    if generator is not None:
        generator.set_state(st)
    else:
        torch.set_rng_state(st)
    return out


_rng_replay_ok = None


def torch_rng_replay_ok() -> bool:
    """One-time self-check of the native replay against torch itself (private generators, a skip that crosses
    blocks, the reference's uniform range).  False -> callers use torch's own operators (slower, same numbers)."""
    global _rng_replay_ok
    if _rng_replay_ok is None:
        import torch
        try:
            g1, g2 = torch.Generator(), torch.Generator()
            g1.manual_seed(20240607); g2.manual_seed(20240607)
            torch.empty(1531).uniform_(-0.04, 0.04, generator=g1)
            want = torch.empty(2000).uniform_(1e-5, 1.0 - 1e-5, generator=g1)
            got = torch_rng_uniform(1531, 2000, 1e-5, 1.0 - 1e-5, generator=g2)
            tail_w = torch.empty(700).uniform_(generator=g1)
            tail_g = torch.empty(700).uniform_(generator=g2)
            ok = torch.equal(want, got) and torch.equal(tail_w, tail_g)
            want2 = torch.empty(40, 55).uniform_(1e-5, 1.0 - 1e-5, generator=g1)
            got2 = torch_rng_uniform(0, 40 * 55, 1e-5, 1.0 - 1e-5, generator=g2, row_len=55, cols=((10, 30), (52, 54)))
            ok = ok and torch.equal(torch.cat([want2[:, 10:30], want2[:, 52:54]], 1).reshape(-1), got2)
            ok = ok and torch.equal(torch.empty(5).uniform_(generator=g1), torch.empty(5).uniform_(generator=g2))
            _rng_replay_ok = bool(ok)
        except Exception:
            _rng_replay_ok = False
    return _rng_replay_ok
