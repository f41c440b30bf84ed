"""Drop-in replacement for the reference's utils/dsp.py, for environments where librosa 0.6.3 does not install: copy THIS
file over `utils/dsp.py` of a reference checkout (the repository root of wavernn-b200 on PYTHONPATH).  It re-exports
wavernn_b200/dropin_dsp.py, whose `hp` is the checkout's own utils.hparams."""
from wavernn_b200.dropin_dsp import *  # noqa: F401,F403
