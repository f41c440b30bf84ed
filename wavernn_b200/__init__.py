"""wavernn_b200 -- Hopper (sm_90a) native WaveRNN batched vocoder.

One hot path, behind the reference's own Python surface:

    from wavernn_b200 import WaveRNN           # same ctor / state_dict / generate()
    model.generate(mels, save_path, batched, target, overlap, mu_law)

The sample-by-sample loop of fatchord/WaveRNN `models/fatchord_version.py:201-241`
runs as ONE persistent CUDA kernel (wavernn_b200/csrc) reached through a C-ABI
shared library (include/wavernn_b200.h).  There is no CPU fallback: without the
built library or without a CUDA device `generate()` raises.
"""
from .hp import hparams  # noqa: F401
from .vocoder import WaveRNN, UpsampleNetwork, MelResNet, ResBlock, Stretch2d  # noqa: F401

__all__ = ["WaveRNN", "UpsampleNetwork", "MelResNet", "ResBlock", "Stretch2d", "hparams"]
__version__ = "0.1.0"
