"""Drop-in replacement for the reference's models/fatchord_version.py (fatchord/WaveRNN @ 83c08fd).

Copy THIS file over `models/fatchord_version.py` of a reference checkout (the repository root of wavernn-b200 on
PYTHONPATH) and `gen_wavernn.py`, `gen_tacotron.py`, `quick_start.py` and `train_wavernn.py` run unchanged:
they only touch `WaveRNN(**hp...)`, `.to(device)`, `.load(path)`, `.get_step()`, `.generate(mels, save_path, batched,
target, overlap, mu_law)` and, for training, `.forward(x, mels)` (gen_wavernn.py:112-137, gen_tacotron.py:78-92,139-163,
quick_start.py:53-64,120, train_wavernn.py:54-65).  Same constructor, same 148 state_dict keys, same return value and
wav side effect; the per-sample loop (:201-241) is the persistent sm_90a kernel behind include/wavernn_b200.h.
Without a file swap: `python -m wavernn_b200.dropin gen_wavernn.py ...` injects the same module at import time.
"""
from wavernn_b200.vocoder import MelResNet, ResBlock, Stretch2d, UpsampleNetwork, WaveRNN  # noqa: F401
