"""The `utils.dsp` stand-in of `python -m wavernn_b200.dropin`, on a minimal fake reference checkout: served only where
librosa cannot be found, executed when the script imports it (its `hp` is the checkout's own singleton), exporting what
the reference's scripts read through `from utils.dsp import *`, and loading a WAV at the model's rate bit-exactly
without a GPU."""
import importlib.util
import json
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent

# what gen_wavernn.py, gen_tacotron.py, preprocess.py and utils/dataset.py read from utils.dsp
EXPORTS = ("hp", "np", "math", "load_wav", "save_wav", "melspectrogram", "reconstruct_waveform", "label_2_float",
           "float_2_label", "encode_mu_law", "decode_mu_law", "normalize", "denormalize", "amp_to_db", "db_to_amp",
           "split_signal", "combine_signal", "encode_16bits", "pre_emphasis", "de_emphasis")

HPARAMS = """sample_rate = 22050
n_fft = 2048
num_mels = 80
hop_length = 275
win_length = 1100
fmin = 40
min_level_db = -100
ref_level_db = 20
preemphasis = 0.97
"""

# the checkout's hparams singleton: configured once, from a python file, after the scripts' imports
UTILS_INIT = """import importlib.util


class _HParams:
    def configure(self, path):
        spec = importlib.util.spec_from_file_location("hparams", path)
        m = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(m)
        for k, v in vars(m).items():
            if not k.startswith("__"):
                setattr(self, k, v)


hparams = _HParams()
"""

OWN_DSP = """import librosa
SOURCE = "checkout"
"""

SCRIPT = """import json
import sys

from utils.dsp import *
import utils
import utils.dsp as D

utils.hparams.configure("hparams.py")
out = {"file": D.__file__, "names": sorted(k for k in globals() if not k.startswith("_")),
       "hp_is_checkout": globals().get("hp") is utils.hparams, "standin": getattr(D, "SOURCE", "standin")}
if out["standin"] == "standin":
    import torch
    out["cuda_initialised"] = torch.cuda.is_initialized()
    cabi = sys.modules.get("wavernn_b200.cabi")
    out["library_loaded"] = cabi is not None and cabi._lib is not None
    mode = sys.argv[1]
    if mode != "import":
        y = load_wav(sys.argv[2])
        np.save("loaded.npy", y)
        if mode == "mel":
            np.save("mel.npy", melspectrogram(y))
json.dump(out, open("result.json", "w"))
"""


def make_checkout(root: Path):
    (root / "utils").mkdir(parents=True)
    (root / "utils" / "__init__.py").write_text(UTILS_INIT)
    (root / "utils" / "dsp.py").write_text(OWN_DSP)
    (root / "hparams.py").write_text(HPARAMS)
    (root / "script.py").write_text(SCRIPT)


def run_dropin(root: Path, *args, extra_path=()):
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([*map(str, extra_path), str(ROOT)] + ([env["PYTHONPATH"]] if env.get("PYTHONPATH") else []))
    r = subprocess.run([sys.executable, "-m", "wavernn_b200.dropin", "script.py", *args], cwd=root, env=env,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    return json.loads((root / "result.json").read_text())


def write_wav16(path, data, sr):
    from scipy.io import wavfile
    wavfile.write(str(path), sr, data.astype(np.int16))


def librosa_decode16(data):
    """librosa 0.6.3's load of 16-bit PCM before resampling: buf_to_float (int16 * 2^-15 in float32) on the interleaved
    samples, reshaped to [channels, n], then to_mono's np.mean over channels."""
    y = (1.0 / 32768) * data.reshape(-1).astype(np.float32)
    y = y.reshape((-1, data.shape[1])).T
    return np.mean(y, axis=0)


needs_no_librosa = pytest.mark.skipif(importlib.util.find_spec("librosa") is not None,
                                      reason="librosa is importable here, so the checkout's own utils.dsp is served")


@needs_no_librosa
def test_standin_exports_and_binds_checkout_hp(tmp_path):
    make_checkout(tmp_path)
    out = run_dropin(tmp_path, "import")
    assert out["standin"] == "standin"
    assert Path(out["file"]).resolve() == (ROOT / "wavernn_b200" / "dropin_dsp.py").resolve()
    assert not set(EXPORTS) - set(out["names"])
    assert out["hp_is_checkout"]
    assert not out["cuda_initialised"] and not out["library_loaded"]


@needs_no_librosa
def test_same_rate_stereo_wav_loads_bit_exactly(tmp_path):
    make_checkout(tmp_path)
    rs = np.random.RandomState(0)
    data = rs.randint(-32768, 32768, size=(5000, 2)).astype(np.int16)
    data[:3] = [[-32768, -32768], [32767, 32767], [-32768, 32767]]
    write_wav16(tmp_path / "a.wav", data, 22050)
    out = run_dropin(tmp_path, "load", str(tmp_path / "a.wav"))
    assert not out["cuda_initialised"] and not out["library_loaded"]
    y = np.load(tmp_path / "loaded.npy")
    want = librosa_decode16(data)
    assert y.dtype == np.float32 and np.array_equal(y.view(np.int32), want.view(np.int32))


def test_checkout_dsp_used_when_librosa_is_found(tmp_path):
    make_checkout(tmp_path / "checkout")
    fake = tmp_path / "site"
    (fake / "librosa").mkdir(parents=True)
    (fake / "librosa" / "__init__.py").write_text("")
    out = run_dropin(tmp_path / "checkout", "import", extra_path=[fake])
    assert out["standin"] == "checkout"
    assert Path(out["file"]).resolve() == (tmp_path / "checkout" / "utils" / "dsp.py").resolve()


def test_standin_helpers():
    """The helpers that need no device, against their definitions."""
    import types
    hp = types.SimpleNamespace(min_level_db=-100, preemphasis=0.97)
    fake_utils = types.ModuleType("utils")
    fake_utils.hparams = hp
    saved = sys.modules.get("utils")
    sys.modules["utils"] = fake_utils
    try:
        spec = importlib.util.spec_from_file_location("standin_dsp_under_test", ROOT / "wavernn_b200" / "dropin_dsp.py")
        D = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(D)
    finally:
        if saved is None:
            del sys.modules["utils"]
        else:
            sys.modules["utils"] = saved
    assert D.hp is hp
    x = np.array([-32768, -1, 0, 255, 256, 32767])
    c, f = D.split_signal(x)
    assert np.array_equal(c, (x + 32768) // 256) and np.array_equal(f, (x + 32768) % 256)
    assert np.array_equal(D.combine_signal(c, f), x)
    assert np.array_equal(D.encode_16bits(np.array([-2.0, -1.0, 0.5, 1.0])), np.array([-32768, -32768, 16384, 32767]))
    S = np.array([-120.0, -100.0, -50.0, 0.0, 10.0])
    assert np.allclose(D.normalize(S), [0, 0, 0.5, 1, 1])
    assert np.allclose(D.denormalize(D.normalize(S)), [-100, -100, -50, 0, 0])
    assert np.allclose(D.db_to_amp(D.amp_to_db(np.array([1e-6, 1e-3, 0.5]))), [1e-5, 1e-3, 0.5])
    rs = np.random.RandomState(1)
    s = rs.randn(100)
    e = D.pre_emphasis(s)
    assert np.allclose(e[1:], s[1:] - 0.97 * s[:-1]) and np.allclose(D.de_emphasis(e), s)
