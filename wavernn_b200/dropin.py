"""Run an UNMODIFIED reference CLI (gen_wavernn.py, gen_tacotron.py, quick_start.py, train_wavernn.py) with the H100
vocoder underneath:

    cd /path/to/WaveRNN && python -m wavernn_b200.dropin gen_wavernn.py --file mel.npy --batched

The scripts reach the vocoder only through `from models.fatchord_version import WaveRNN` (gen_wavernn.py:3,
gen_tacotron.py:2, quick_start.py:2, train_wavernn.py:8).  `install()` registers a module of that name -- the same
re-export as dropin/models/fatchord_version.py -- in sys.modules before the script is executed, so the import resolves
to wavernn_b200.vocoder while `models.tacotron`, `utils.*`, `hparams.py` and the checkpoints stay the reference's own.
Nothing in the reference checkout is modified.

The one exception to `utils.*`: where librosa cannot be imported, the reference's utils/dsp.py (which imports it on its
first line, and which gen_wavernn.py, gen_tacotron.py, preprocess.py and utils/dataset.py import) cannot run, so
`install()` also serves `utils.dsp` from wavernn_b200/dropin_dsp.py.  Where librosa imports, the checkout's own module
is used, as before.
"""
from __future__ import annotations

import importlib.abc
import importlib.util
import os
import runpy
import sys
import types

SHIM_NAME = "models.fatchord_version"
EXPORTS = ("WaveRNN", "UpsampleNetwork", "MelResNet", "ResBlock", "Stretch2d")
DSP_NAME = "utils.dsp"
DSP_SOURCE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "dropin_dsp.py")


class DspFinder(importlib.abc.MetaPathFinder):
    """Finds `utils.dsp` as wavernn_b200/dropin_dsp.py, executed under that name when the script first imports it (so
    its `from utils import hparams` binds the checkout's singleton)."""

    def find_spec(self, fullname, path=None, target=None):
        return importlib.util.spec_from_file_location(DSP_NAME, DSP_SOURCE) if fullname == DSP_NAME else None


def install() -> types.ModuleType:
    """Registers the replacement `models.fatchord_version` and, when librosa cannot be found, the `utils.dsp` stand-in
    (idempotent).  Returns the `models.fatchord_version` module."""
    if importlib.util.find_spec("librosa") is None and not any(isinstance(f, DspFinder) for f in sys.meta_path):
        sys.meta_path.insert(0, DspFinder())
    from . import vocoder
    mod = sys.modules.get(SHIM_NAME)
    if mod is not None and getattr(mod, "__wavernn_b200__", False):
        return mod
    mod = types.ModuleType(SHIM_NAME, "wavernn_b200 drop-in for the reference's models/fatchord_version.py")
    for name in EXPORTS:
        setattr(mod, name, getattr(vocoder, name))
    mod.__wavernn_b200__ = True
    mod.__file__ = vocoder.__file__
    sys.modules[SHIM_NAME] = mod
    return mod


def main(argv=None) -> int:
    argv = list(sys.argv[1:] if argv is None else argv)
    if not argv or argv[0] in ("-h", "--help"):
        print(__doc__)
        return 0 if argv else 2
    script = os.path.abspath(argv[0])
    if not os.path.isfile(script):
        print(f"wavernn_b200.dropin: no such script: {argv[0]}", file=sys.stderr)
        return 2
    script_dir = os.path.dirname(script)
    if script_dir in sys.path:
        sys.path.remove(script_dir)
    sys.path.insert(0, script_dir)          # what `python script.py` does: the script's packages (models/, utils/) win
    install()
    sys.argv = [script] + argv[1:]
    runpy.run_path(script, run_name="__main__")
    return 0


if __name__ == "__main__":
    sys.exit(main())
